"""GPU: the staged 4-bit GEMM route, the large-M form of path 1 -- each weight panel decoded once into the
per-stream workspace, then the wgmma GEMM with both operands in shared memory.

Its weights are the fused kernel's bit for bit (the same table decode and scale fetch), the k16 order, instruction
shape and epilogue rounding are the same, so its output must equal the fused kernel's (cbnb_b200_gemm_4bit_pair
without a K split) exactly, at both token tiles, for any panel size, and stay within the double-precision oracle's
bounds."""
import ctypes as ct

import pytest
import torch

from tests import _native as nat
from tests.test_gpu_gemm4 import assert_close_to_exact, exact, make_problem

pytestmark = pytest.mark.gpu



def takes_route(M, N, K, dtype_id, bs=64):
    return nat.lib.cbnb_b200_gemm_4bit_staged_route(M, N, K, bs, dtype_id) == 1


def fused(p, mt, out=None, ldc=None):
    M, N, K = p["M"], p["N"], p["K"]
    if out is None:
        out = torch.full((M, N), float("nan"), device="cuda", dtype=nat.DTYPE[p["dtype"]])
    rc = nat.lib.cbnb_b200_gemm_4bit_pair(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
        nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]), nat.ptr(out), nat.ptr(p["bias"]), M, N, K,
        ldc or N, p["bs"], nat.QT_ID[p["qt"]], nat.DTYPE_ID[p["dtype"]], mt, 1, None, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    return out


def staged(p, mt, panel_rows, outs=None, ldc=None):
    M, N, K = p["M"], p["N"], p["K"]
    if outs is None:
        outs = [torch.full((M, N), float("nan"), device="cuda", dtype=nat.DTYPE[p["dtype"]])]
    ptrs = (ct.c_void_p * len(outs))(*[o if isinstance(o, int) else o.data_ptr() for o in outs])
    rc = nat.lib.cbnb_b200_gemm_4bit_staged(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
        nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]), ct.cast(ptrs, ct.c_void_p), len(outs),
        nat.ptr(p["bias"]), M, N, K, ldc or N, p["bs"], nat.QT_ID[p["qt"]], nat.DTYPE_ID[p["dtype"]], mt, panel_rows,
        nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    return outs[0]


def same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# (M, N, K, qt, dtype, blocksize, nested, bias, panel_rows): M tails, N tails (N % 128 != 0), panel tails, rows that
# begin inside a quantisation block (K = 576 at blocksize 128, K = 704 at blocksize 4096), K = 64, several panels
CASES = [
    (300, 384, 512, "nf4", "bf16", 64, True, True, 128),
    (515, 520, 576, "fp4", "fp16", 128, False, True, 256),
    (257, 256, 64, "nf4", "fp16", 32, False, False, 128),
    (640, 1000, 704, "fp4", "bf16", 4096, False, True, 384),
    (1100, 1024, 1024, "nf4", "bf16", 64, True, False, 0),
    (333, 768, 256, "fp4", "fp16", 64, True, True, 256),
    (200, 512, 512, "nf4", "bf16", 128, True, True, 128),
    (129, 640, 576, "nf4", "fp16", 32, False, True, 512),
]


@pytest.mark.parametrize("M,N,K,qt,dtype,bs,nested,bias,panel", CASES)
def test_staged_equals_fused_kernel_bit_for_bit(M, N, K, qt, dtype, bs, nested, bias, panel):
    p = make_problem(M, N, K, qt, dtype, bs=bs, nested=nested, bias=bias, seed=31)
    y64 = exact(p)
    for mt in (128, 256):
        want = fused(p, mt)
        got = staged(p, mt, panel)
        assert same_bits(got, want), f"mt={mt}: staged route differs from the fused kernel"
        assert_close_to_exact(got, y64, dtype, K)
    # the automatic token tile and the default panel give the same bits
    assert same_bits(staged(p, 0, 0), want)


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_staged_strided_unaligned_and_multi_destination_outputs(dtype):
    M, N, K, NF, col0 = 777, 640, 512, 1280, 384
    p = make_problem(M, N, K, "nf4", dtype, bias=True, seed=32)
    want = fused(p, 256)
    bufs = [torch.full((M, NF), -7.0, dtype=nat.DTYPE[dtype], device="cuda") for _ in range(3)]
    staged(p, 256, 256, outs=[b.data_ptr() + col0 * 2 for b in bufs], ldc=NF)
    for b in bufs:
        assert same_bits(b[:, col0:col0 + N].contiguous(), want)
        assert (b[:, :col0] == -7.0).all() and (b[:, col0 + N:] == -7.0).all()
    # a row pitch that is not a multiple of 16 bytes: the element-wise store
    odd = torch.full((M, N + 3), -7.0, dtype=nat.DTYPE[dtype], device="cuda")
    staged(p, 128, 128, outs=[odd], ldc=N + 3)
    assert same_bits(odd[:, :N].contiguous(), want) and (odd[:, N:] == -7.0).all()


@pytest.mark.parametrize("qt,dtype,bs", [("nf4", "bf16", 64), ("fp4", "fp16", 32), ("nf4", "fp16", 4096)])
def test_decoded_panel_equals_dequantize_4bit(qt, dtype, bs):
    """A panel at a non-zero row offset, nested statistics: the same bits as the same rows of F.dequantize_4bit."""
    import bitsandbytes_b200.functional as F

    N, K, n0, rows = 1536, 576, 256, 700
    g = torch.Generator(device="cpu").manual_seed(33)
    W = torch.randn(N, K, generator=g).to(nat.DTYPE[dtype]).cuda()
    qW, qs = F.quantize_4bit(W, blocksize=bs, quant_type=qt, compress_statistics=True)
    want = F.dequantize_4bit(qW, qs)
    out = torch.full((rows, K), float("nan"), device="cuda", dtype=nat.DTYPE[dtype])
    off = qs.offset.to(torch.float32).reshape(1).contiguous()
    rc = nat.lib.cbnb_b200_dequantize_4bit_panel(
        qW.data_ptr(), qs.state2.absmax.data_ptr(), qs.absmax.data_ptr(), qs.state2.code.data_ptr(), off.data_ptr(),
        out.data_ptr(), bs, nat.QT_ID[qt], nat.DTYPE_ID[dtype], n0, rows, K, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    assert same_bits(out, want.view(N, K)[n0:n0 + rows].contiguous())


def test_routing_of_the_benchmark_shapes():
    path = nat.lib.cbnb_b200_gemm_4bit_path
    for n, k in ((4096, 4096), (11008, 4096), (4096, 11008)):
        assert path(4096, n, k, 64, 2) == 1 and takes_route(4096, n, k, 2), (n, k)
    assert path(1, 4096, 4096, 64, 2) == 0 and not takes_route(1, 4096, 4096, 2)
    assert path(16, 4096, 4096, 64, 2) == 1 and not takes_route(16, 4096, 4096, 2)
    assert path(256, 4096, 4096, 64, 2) == 1 and not takes_route(256, 4096, 4096, 2)
    assert path(4096, 4096, 4096, 64, 3) == 1 and not takes_route(4096, 4096, 4096, 3)  # fp32 on TF32
    # a forced path 1 keeps the fused kernel
    nat.lib.cbnb_b200_gemm_4bit_force_path(1)
    try:
        assert not takes_route(4096, 4096, 4096, 2)
    finally:
        nat.lib.cbnb_b200_gemm_4bit_force_path(-1)


def test_matmul_4bit_and_multi_out_take_the_route_with_the_fused_kernels_bits():
    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    M, N, K = 2048, 4096, 1024
    assert takes_route(M, N, K, 2)
    torch.manual_seed(34)
    W = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="nf4", compress_statistics=True)
    got = bnb.matmul_4bit(x, qW.t(), qs)
    nat.lib.cbnb_b200_gemm_4bit_force_path(1)
    try:
        want = bnb.matmul_4bit(x, qW.t(), qs)
    finally:
        nat.lib.cbnb_b200_gemm_4bit_force_path(-1)
    torch.cuda.synchronize()
    assert same_bits(got, want)
    # the fused all-gather entry takes the same route for the same shape: every destination holds the same bits
    bufs = [torch.zeros(M, N, device="cuda", dtype=torch.bfloat16) for _ in range(2)]
    ptrs = (ct.c_void_p * 2)(*[b.data_ptr() for b in bufs])
    off = qs.offset.to(torch.float32).reshape(1).contiguous()
    rc = nat.lib.cbnb_b200_gemm_4bit_multi_out(
        x.data_ptr(), qW.data_ptr(), qs.state2.absmax.data_ptr(), qs.absmax.data_ptr(), qs.state2.code.data_ptr(),
        off.data_ptr(), ct.cast(ptrs, ct.c_void_p), 2, None, M, N, K, N, 64, nat.QT_ID["nf4"], 2, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    assert same_bits(bufs[0], want) and same_bits(bufs[1], want)


def test_cuda_graph_capture_and_two_streams():
    """The workspace is first requested inside the capture (a fresh stream); replay equals eager; two streams at
    once each use their own workspace."""
    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    M, N, K = 2048, 4096, 512
    torch.manual_seed(35)
    W = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.float16)
    qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="fp4")
    xs = [torch.randn(M, K, device="cuda", dtype=torch.float16) for _ in range(2)]
    assert takes_route(M, N, K, 1)
    eager = [bnb.matmul_4bit(x, qW.t(), qs) for x in xs]
    torch.cuda.synchronize()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        y = bnb.matmul_4bit(xs[0], qW.t(), qs)
    graph.replay()
    torch.cuda.synchronize()
    assert same_bits(y, eager[0])

    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for st in (s1, s2):
        st.wait_stream(torch.cuda.current_stream())
    outs = []
    for _ in range(3):
        with torch.cuda.stream(s1):
            a = bnb.matmul_4bit(xs[0], qW.t(), qs)
        with torch.cuda.stream(s2):
            b = bnb.matmul_4bit(xs[1], qW.t(), qs)
        outs.append((a, b))
    torch.cuda.synchronize()
    for a, b in outs:
        assert same_bits(a, eager[0]) and same_bits(b, eager[1])


def test_options_the_route_does_not_serve_are_refused():
    p = make_problem(256, 256, 128, "nf4", "bf16", seed=36)
    out = torch.empty(256, 256, device="cuda", dtype=torch.bfloat16)
    ptrs = (ct.c_void_p * 1)(out.data_ptr())
    base = (nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), None, None, None, ct.cast(ptrs, ct.c_void_p), 1,
            None, 256, 256, 128, 256, 64, nat.QT_ID["nf4"])
    st = nat.stream()
    assert nat.lib.cbnb_b200_gemm_4bit_staged(*base, 2, 64, 0, st) == 100     # token tile 64
    assert nat.lib.cbnb_b200_gemm_4bit_staged(*base, 2, 0, 100, st) == 100    # panel not a multiple of 128
    assert nat.lib.cbnb_b200_gemm_4bit_staged(*base, 0, 0, 0, st) == 100      # fp32
    nat.check()
