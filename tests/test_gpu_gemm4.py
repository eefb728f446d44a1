"""GPU parity: the 4-bit dequant-fused GEMM (wgmma and CUDA-core paths) through the C ABI.

Oracle: oracle/oracle_c.c::oracle_gemm_4bit -- exactly-rounded weights
W_T = rn_T(value * scale), double-precision accumulation.  Tolerance (BASELINE.json
north_star: "<= 1e-3 rel for bf16 GEMM outputs"): the kernels accumulate the same
products in fp32 (tensor cores) and round once to T, so

    |ours - exact| <= ulp_T(exact)/2 + fp32 accumulation error
    rel_fro(ours, rn_T(exact)) <= 1e-3            (measured ~2e-4..4e-4 for bf16: rounding flips)

and against the reference CUDA library on the same buffers the same two bounds hold with
`exact` replaced by the reference's output (its accumulation order differs).
"""
import numpy as np
import pytest
import torch

import oracle
from tests import _native as nat

pytestmark = pytest.mark.gpu

MANT_BITS = {"bf16": 7, "fp16": 10, "fp32": 23}  # explicit significand bits of T


def make_problem(M, N, K, qt, dtype, bs=64, nested=False, bias=False, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed * 7919 + M * 31 + N * 17 + K)
    W = (torch.randn(N, K, generator=g) / K**0.5).to(nat.DTYPE[dtype]).cuda()
    x = torch.randn(M, K, generator=g).to(nat.DTYPE[dtype]).cuda()
    packed, absmax = nat.quantize(nat.lib, W.view(-1), bs, qt, None, dtype)
    p = dict(x=x, packed=packed, absmax=absmax, M=M, N=N, K=K, bs=bs, qt=qt, dtype=dtype, bias=None,
             absmax_8bit=None, absmax_code=None, absmax_offset=None)
    if nested:
        from bitsandbytes_b200.functional import create_dynamic_map

        code2 = create_dynamic_map().cuda()
        offset = absmax.mean().reshape(1)
        a8, a2 = nat.quantize(nat.lib, (absmax - offset).contiguous(), 256, None, code2, "fp32")
        p.update(absmax=a2, absmax_8bit=a8, absmax_code=code2, absmax_offset=offset)
    if bias:
        p["bias"] = torch.randn(N, generator=g).to(nat.DTYPE[dtype]).cuda()
    return p


def run(L, p):
    return nat.gemm_4bit(L, p["x"], p["packed"], p["absmax"], p["M"], p["N"], p["K"], p["bs"], p["qt"], p["dtype"],
                         p["bias"], p["absmax_8bit"], p["absmax_code"], p["absmax_offset"])


def exact(p):
    dt = p["dtype"]
    x = oracle.widen(nat.to_bits(p["x"]), dt)
    bias = oracle.widen(nat.to_bits(p["bias"]), dt) if p["bias"] is not None else None
    kw = {}
    if p["absmax_8bit"] is not None:
        kw = dict(absmax_8bit=p["absmax_8bit"].cpu().numpy(), absmax_code=p["absmax_code"].cpu().numpy(),
                  absmax_offset=float(p["absmax_offset"].item()))
    return oracle.gemm_4bit(x, p["packed"].cpu().numpy(), p["absmax"].cpu().numpy(), p["M"], p["N"], p["K"], p["bs"],
                            p["qt"], dt, bias, **kw)


def assert_close_to_exact(got: torch.Tensor, y64: np.ndarray, dtype: str, K: int):
    g = got.double().cpu().numpy()
    assert np.all(np.isfinite(g)), "non-finite outputs (unwritten tile?)"
    scale = np.abs(y64)
    # half an ulp of T at the exact value (ulp = 2^(floor(log2|y|) - mant_bits)) + fp32
    # accumulation slack (|terms| ~ O(1/sqrt(K)), K of them)
    ulp = np.exp2(np.floor(np.log2(np.maximum(scale, 1e-30))) - MANT_BITS[dtype])
    tol = 0.5 * ulp * 1.001 + 2.0**-22 * np.sqrt(K) * (1.0 + scale) + 1e-30
    bad = np.abs(g - y64) > tol
    assert not bad.any(), f"{bad.sum()} / {bad.size} outputs off; worst {np.max(np.abs(g - y64) / (scale + 1e-6)):.3e}"
    want = torch.from_numpy(y64).to(got.dtype).double().numpy()
    rel = np.linalg.norm(g - want) / (np.linalg.norm(want) + 1e-30)
    assert rel <= 1e-3, rel


SHAPES_SMALL = [
    (1, 128, 64), (1, 256, 4096), (3, 130, 128), (5, 48, 128), (16, 128, 256), (17, 384, 512),
    (33, 200, 192), (64, 128, 1024), (100, 256, 128), (128, 512, 256), (200, 128, 320), (256, 256, 512),
    (300, 384, 128), (513, 128, 64),
]


@pytest.mark.parametrize("path", [1, 0], ids=["tcgen05", "simt"])
@pytest.mark.parametrize("M,N,K", SHAPES_SMALL)
def test_bf16_nf4_vs_oracle(path, M, N, K):
    p = make_problem(M, N, K, "nf4", "bf16")
    nat.lib.cbnb_b200_gemm_4bit_force_path(path)
    try:
        got = run(nat.lib, p)
    finally:
        nat.lib.cbnb_b200_gemm_4bit_force_path(-1)
    nat.check()
    assert_close_to_exact(got, exact(p), "bf16", K)


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("nested,bias,bs", [(False, True, 64), (True, False, 64), (True, True, 128), (False, False, 32),
                                            (False, True, 256)])
def test_variants_vs_oracle(dtype, qt, nested, bias, bs):
    # N*K/bs must be a multiple of 256 for the nested case (double-quant blocks of 256 absmax values)
    M, N, K = 37, 512, 256
    p = make_problem(M, N, K, qt, dtype, bs=bs, nested=nested, bias=bias, seed=3)
    for path in (1, 0):
        nat.lib.cbnb_b200_gemm_4bit_force_path(path)
        try:
            got = run(nat.lib, p)
        finally:
            nat.lib.cbnb_b200_gemm_4bit_force_path(-1)
        nat.check()
        assert_close_to_exact(got, exact(p), dtype, K)


# the mma.sync decode kernel (path 3): every M it serves, ragged N, K tails inside a 256-wide chunk,
# blocksize 32 (two scales per lane) up to blocksize > chunk, both dtypes / code books, nested, bias
@pytest.mark.parametrize("M,N,K", [(1, 128, 64), (1, 4096, 4096), (2, 130, 128), (5, 48, 320), (8, 16, 256),
                                   (7, 40, 704), (6, 384, 512), (8, 1000, 1024), (8, 14336, 512)])
def test_decode_kernel_vs_oracle(M, N, K):
    p = make_problem(M, N, K, "nf4", "bf16")
    assert nat.lib.cbnb_b200_gemm_4bit_path(M, N, K, p["bs"], 2) in (0, 3)
    nat.lib.cbnb_b200_gemm_4bit_force_path(3)
    try:
        got = run(nat.lib, p)
    finally:
        nat.lib.cbnb_b200_gemm_4bit_force_path(-1)
    nat.check()
    assert_close_to_exact(got, exact(p), "bf16", K)


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("nested,bias,bs", [(False, True, 64), (True, False, 64), (True, True, 128), (False, False, 32),
                                            (False, True, 512)])
def test_decode_kernel_variants_vs_oracle(dtype, qt, nested, bias, bs):
    M, N, K = 7, 512, 768
    p = make_problem(M, N, K, qt, dtype, bs=bs, nested=nested, bias=bias, seed=4)
    nat.lib.cbnb_b200_gemm_4bit_force_path(3)
    try:
        got = run(nat.lib, p)
    finally:
        nat.lib.cbnb_b200_gemm_4bit_force_path(-1)
    nat.check()
    assert_close_to_exact(got, exact(p), dtype, K)


def test_decode_kernel_weights_match_the_tensor_core_path():
    """Same decoded weights, exact products: the two tensor-core paths may differ only by fp32 summation order."""
    p = make_problem(8, 256, 2048, "nf4", "bf16", seed=9)
    outs = []
    for path in (3, 1):
        nat.lib.cbnb_b200_gemm_4bit_force_path(path)
        try:
            outs.append(run(nat.lib, p).float())
        finally:
            nat.lib.cbnb_b200_gemm_4bit_force_path(-1)
    nat.check()
    assert torch.allclose(outs[0], outs[1], rtol=2e-2, atol=1e-3)
    assert (outs[0] - outs[1]).abs().max().item() <= 2.0 ** -6 * outs[1].abs().max().item()


@pytest.mark.parametrize("M,N,K", [(1, 64, 96), (4, 100, 72), (7, 33, 200)])
def test_fp32_and_odd_shapes_take_the_cuda_core_path(M, N, K):
    p = make_problem(M, N, K, "nf4", "fp32", bs=64 if (N * K) % 64 == 0 else 32)
    assert nat.lib.cbnb_b200_gemm_4bit_path(M, N, K, p["bs"], 0) == 2
    got = run(nat.lib, p)
    nat.check()
    assert_close_to_exact(got, exact(p), "fp32", K)


def test_split_k_is_deterministic_and_workspace_self_resets():
    p = make_problem(8, 256, 4096, "nf4", "bf16", seed=5)
    a = run(nat.lib, p)
    b = run(nat.lib, p)
    c = run(nat.lib, p)
    assert torch.equal(a, b) and torch.equal(b, c)
    assert_close_to_exact(a, exact(p), "bf16", 4096)


def test_multi_destination_epilogue_writes_every_buffer():
    """The fused all-gather epilogue on one GPU: three 'peer' buffers on the same device must all receive
    this shard's columns, bit-identical to the plain call, and nothing else may be touched."""
    import ctypes as ct

    M, N, K, NF = 300, 256, 512, 1024  # shard of 256 features at column 384 of a 1024-wide output
    p = make_problem(M, N, K, "nf4", "bf16", bias=True, seed=11)
    want = run(nat.lib, p)
    bufs = [torch.full((M, NF), -7.0, dtype=torch.bfloat16, device="cuda") for _ in range(3)]
    col0 = 384
    ptrs = (ct.c_void_p * 3)(*[b.data_ptr() + col0 * 2 for b in bufs])
    rc = nat.lib.cbnb_b200_gemm_4bit_multi_out(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), None, None, None, ct.cast(ptrs, ct.c_void_p), 3,
        nat.ptr(p["bias"]), M, N, K, NF, p["bs"], nat.QT_ID["nf4"], 2, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    for b in bufs:
        assert torch.equal(b[:, col0:col0 + N], want)
        assert (b[:, :col0] == -7.0).all() and (b[:, col0 + N:] == -7.0).all()
    # split-K shapes take the cooperative reduction: same contract
    M2 = 24
    p2 = make_problem(M2, N, 4096, "nf4", "bf16", seed=12)
    nat.lib.cbnb_b200_gemm_4bit_force_path(1)
    try:
        want2 = run(nat.lib, p2)
    finally:
        nat.lib.cbnb_b200_gemm_4bit_force_path(-1)
    bufs2 = [torch.zeros((M2, N), dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    ptrs2 = (ct.c_void_p * 2)(*[b.data_ptr() for b in bufs2])
    rc = nat.lib.cbnb_b200_gemm_4bit_multi_out(
        nat.ptr(p2["x"]), nat.ptr(p2["packed"]), nat.ptr(p2["absmax"]), None, None, None, ct.cast(ptrs2, ct.c_void_p),
        2, None, M2, N, 4096, N, p2["bs"], nat.QT_ID["nf4"], 2, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    assert torch.equal(bufs2[0], want2) and torch.equal(bufs2[1], want2)
    # fp32 activations do not take the tensor-core kernel: the entry point says so instead of computing
    assert nat.lib.cbnb_b200_gemm_4bit_multi_out(None, None, None, None, None, None, ct.cast(ptrs2, ct.c_void_p), 2,
                                                 None, M2, N, 4096, N, 64, nat.QT_ID["nf4"], 0, nat.stream()) == 100


def test_strided_output_for_sharded_linear():
    p = make_problem(32, 256, 256, "nf4", "bf16", seed=9)
    full = torch.zeros(32, 1024, device="cuda", dtype=torch.bfloat16)
    view = full[:, 512:768]
    nat.lib.cbnb_b200_gemm_4bit_strided(p["x"].data_ptr(), p["packed"].data_ptr(), p["absmax"].data_ptr(), None, None,
                                        None, view.data_ptr(), None, 32, 256, 256, 1024, 64, 2, 2, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert torch.equal(view, run(nat.lib, p))
    assert full[:, :512].abs().sum().item() == 0 and full[:, 768:].abs().sum().item() == 0


@pytest.mark.parametrize("M", [1, 16, 256, 4096])
@pytest.mark.parametrize("N,K", [(4096, 4096), (11008, 4096), (4096, 11008)])
def test_baseline_shapes_vs_reference_cuda_and_dequant_matmul(M, N, K):
    """C2 shapes at full size.  Property: fused GEMM == (our bit-exact dequantize) @ x in fp32 up to
    accumulation order; plus the reference CUDA library's own output on the same buffers."""
    p = make_problem(M, N, K, "nf4", "bf16", seed=11)
    got = run(nat.lib, p)
    nat.check()
    W = nat.dequantize(nat.lib, p["packed"], p["absmax"], 64, N * K, "nf4", None, "bf16").view(N, K)
    want32 = p["x"].float() @ W.float().t()  # fp32 reference of the same op (test-only library call)
    want = want32.to(torch.bfloat16)
    diff = (got.float() - want32).abs()
    tol = want32.abs() * (2.0**-8 * 1.01) + 2.0**-20 * (K**0.5) * (1 + want32.abs())  # half ulp of bf16 <= 2^-8 |y|
    assert (diff <= tol).all(), f"max excess {(diff - tol).max().item():.3e}"
    rel = (got.float() - want.float()).norm() / want.float().norm()
    assert rel.item() <= 1e-3
    ref = nat.ref_cuda()
    if ref is not None:
        r = run(ref, p)
        rel_ref = (got.float() - r.float()).norm() / r.float().norm()
        # M <= 3 takes the reference's SIMT kernel, which rounds every product to bf16
        # (reference gemm_4bit_simt.cu:353,452): compare error-vs-exact instead of each other.
        if M <= 3:
            e_ours = (got.float() - want32).norm()
            e_ref = (r.float() - want32).norm()
            assert e_ours <= e_ref * 1.05 + 1e-6
        else:
            assert rel_ref.item() <= 1e-3, rel_ref.item()


def test_legacy_gemv_entry_point():
    from bitsandbytes_b200.functional import get_4bit_type

    p = make_problem(1, 256, 512, "nf4", "bf16", seed=2)
    code = get_4bit_type("nf4", device="cuda")
    out = torch.zeros(256, device="cuda", dtype=torch.bfloat16)
    nat.lib.cgemm_4bit_inference_naive_bf16(256, 1, 512, p["x"].data_ptr(), p["packed"].data_ptr(),
                                            p["absmax"].data_ptr(), code.data_ptr(), out.data_ptr(), 256, 256, 256, 64,
                                            nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert_close_to_exact(out.view(1, 256), exact(p), "bf16", 512)
