"""GPU: fp32 4-bit GEMMs on TF32 tensor cores, the route taken when PyTorch's fp32 matmul precision is "tf32".

The contract of the route (native dtype 3): weights W = rna_tf32(W32), where W32 is the fp32 weight
``dequantize_4bit(..., float32)`` returns and rna_tf32 rounds to the nearest TF32 value, ties away from zero; the
activations are read as TF32 by the tensor cores; products are accumulated in fp32 and the fp32 bias is added in fp32.
Under the default precision the fp32 route is unchanged, bit for bit.
"""
import numpy as np
import pytest
import torch

import bitsandbytes_b200 as bnb
from bitsandbytes_b200.backends.cuda import gemm_4bit_dtype_id
from tests import _native as nat

pytestmark = pytest.mark.gpu

TF32_MIN_M = 4  # dispatch threshold of dtype 3 (c_api.cu kTf32MinM)


@pytest.fixture
def precision():
    """Sets torch.backends.cuda.matmul.fp32_precision for the test and restores it through the same API."""
    m = torch.backends.cuda.matmul
    prev = m.fp32_precision

    def set_to(value):
        m.fp32_precision = value

    yield set_to
    m.fp32_precision = prev


def tf32_exact(x: torch.Tensor) -> torch.Tensor:
    """x with the 13 low mantissa bits cleared: a value TF32 represents exactly."""
    return (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def rna_tf32(w: torch.Tensor) -> torch.Tensor:
    """Round fp32 to the nearest TF32 value, ties away from zero (cvt.rna.tf32.f32) -- on the sign-magnitude bits."""
    b = w.contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def make_problem(M, N, K, qt="nf4", bs=64, nested=False, bias=False, seed=0, exact_acts=True):
    g = torch.Generator(device="cpu").manual_seed(seed * 7919 + M * 31 + N * 17 + K)
    W = (torch.randn(N, K, generator=g) / K**0.5).cuda()
    x = torch.randn(M, K, generator=g).cuda()
    if exact_acts:
        x = tf32_exact(x)
    packed, absmax = nat.quantize(nat.lib, W.view(-1), bs, qt, None, "fp32")
    p = dict(x=x, packed=packed, absmax=absmax, M=M, N=N, K=K, bs=bs, qt=qt, bias=None, absmax_8bit=None,
             absmax_code=None, absmax_offset=None)
    scale = absmax
    if nested:
        from bitsandbytes_b200.functional import create_dynamic_map

        code2 = create_dynamic_map().cuda()
        offset = absmax.mean().reshape(1)
        a8, a2 = nat.quantize(nat.lib, (absmax - offset).contiguous(), 256, None, code2, "fp32")
        p.update(absmax=a2, absmax_8bit=a8, absmax_code=code2, absmax_offset=offset)
        # the statistics F.dequantize_4bit uses: dequantise the nested absmax, then add the offset (two roundings)
        scale = nat.dequantize(nat.lib, a8, a2, 256, absmax.numel(), None, code2, "fp32") + offset
    if bias:
        p["bias"] = torch.randn(N, generator=g).cuda()
    # W32: the library's bit-exact fp32 dequantisation
    p["W32"] = nat.dequantize(nat.lib, packed, scale.contiguous(), bs, N * K, qt, None, "fp32").view(N, K)
    return p


def native_call(p, dtype_id, x=None):
    """out = x . dequant(B)^T + bias through the strided entry (dispatch of the library) with the given dtype id."""
    x = p["x"] if x is None else x
    M, N, K = x.shape[0], p["N"], p["K"]
    out = torch.full((M, N), float("nan"), device="cuda")
    nat.lib.cbnb_b200_gemm_4bit_strided(
        nat.ptr(x), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]), nat.ptr(p["absmax_code"]),
        nat.ptr(p["absmax_offset"]), nat.ptr(out), nat.ptr(p["bias"]), M, N, K, N, p["bs"], nat.QT_ID[p["qt"]],
        dtype_id, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    return out


def pair_call(p, mt, splits):
    """The TF32 instance with an explicit token tile and K split (developer entry)."""
    M, N, K = p["M"], p["N"], p["K"]
    out = torch.full((M, N), float("nan"), device="cuda")
    rc = nat.lib.cbnb_b200_gemm_4bit_pair(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
        nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]), nat.ptr(out), nat.ptr(p["bias"]), M, N, K, N, p["bs"],
        nat.QT_ID[p["qt"]], 3, mt, splits, None, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0, (mt, splits)
    return out


def op_call(p, x=None):
    x = p["x"] if x is None else x
    off = p["absmax_offset"]
    return torch.ops.bitsandbytes.gemm_4bit(x, p["packed"], [p["N"], p["K"]], p["absmax"], p["bs"], p["qt"], p["bias"],
                                           p["absmax_8bit"], p["absmax_code"], off)


def y64_of(x, W, bias):
    y = x.double() @ W.double().t()
    return y if bias is None else y + bias.double()


def ulp32(y):
    return torch.exp2(torch.floor(torch.log2(y.abs().clamp_min(2.0**-126))) - 23)


def accumulation(K, y64):
    """fp32 accumulation slack: the 2^-22 sqrt(K) term of the 16-bit tests plus 2^-23 per k8 step.  The tensor core does
    not round to nearest when it adds a step's products to the fp32 accumulator, so its error grows with the number of
    steps, not with their square root: at K = 4096 and one K split the outputs measured up to twice the first term."""
    return (2.0**-22 * K**0.5 + 2.0**-23 * (K / 8)) * (1 + y64.abs())


def assert_weights_contract(got, p, x=None):
    """Exact-TF32 activations: every product a * rna_tf32(W32) is exact in fp32, so the outputs differ from the float64
    sum only by half an fp32 ulp and the fp32 accumulation."""
    x = p["x"] if x is None else x
    K = p["K"]
    y64 = y64_of(x.reshape(-1, K), rna_tf32(p["W32"]), p["bias"]).view(got.shape)
    g = got.double()
    assert torch.isfinite(g).all(), "non-finite outputs (unwritten tile?)"
    tol = 0.5 * ulp32(y64) + accumulation(K, y64)
    bad = (g - y64).abs() > tol
    assert not bad.any(), f"{int(bad.sum())} / {bad.numel()} outputs off; worst {float(((g - y64).abs() / tol).max()):.2f} x tol"


def assert_tf32_bound(got, x, W32, bias, what):
    """Arbitrary fp32 activations: TF32 reads them with a relative error below 2^-10 and the weights are rounded with
    one below 2^-11, so |got - y64| <= (2^-10 + 2^-11) sum|a||w| + half an fp32 ulp + the fp32 accumulation."""
    K = x.shape[-1]
    x2 = x.reshape(-1, K)
    y64 = y64_of(x2, W32, bias).view(got.shape)
    s = (x2.double().abs() @ W32.double().abs().t()).view(got.shape)
    tol = (2.0**-10 + 2.0**-11) * (1 + 2.0**-10) * s + 0.5 * ulp32(y64) + accumulation(K, y64)
    g = got.double()
    assert torch.isfinite(g).all(), what
    bad = (g - y64).abs() > tol
    assert not bad.any(), f"{what}: {int(bad.sum())} / {bad.numel()} outputs off"


# ------------------------------------------------------------------------------------------------ 1. default
@pytest.mark.parametrize("M", [16, 4096])
def test_default_precision_is_the_fp32_route_bit_for_bit(precision, M):
    precision("ieee")
    p = make_problem(M, 512, 1024, "nf4", bias=True, seed=1, exact_acts=False)
    assert gemm_4bit_dtype_id(torch.float32) == 0
    assert nat.lib.cbnb_b200_gemm_4bit_path(M, 512, 1024, 64, 0) == 2
    got = op_call(p)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int32), native_call(p, 0).view(torch.int32))


# ------------------------------------------------------------------------------------------------ 2. weights contract
# (M, N, K, qt, blocksize, nested, bias, token tile, forced K split); ragged M and N, K of one, five and 64 stages,
# nested statistics where N * K / blocksize is a multiple of 256
CONTRACT = [
    (16, 256, 64, "nf4", 64, False, False, 16, 1),
    (13, 130, 320, "fp4", 32, False, True, 16, 2),
    (37, 200, 320, "fp4", 32, False, True, 64, 1),
    (33, 256, 320, "fp4", 64, True, True, 32, 2),
    (64, 256, 64, "nf4", 256, False, True, 64, 1),
    (8, 192, 4096, "nf4", 256, True, False, 16, 7),
    (100, 384, 4096, "nf4", 128, True, True, 128, 1),
    (129, 136, 64, "nf4", 32, False, True, 128, 1),
    (300, 512, 4096, "fp4", 256, False, False, 128, 2),
    (50, 1000, 320, "nf4", 64, False, True, 64, 7),
    (200, 264, 4096, "fp4", 128, False, True, 128, 7),
]


@pytest.mark.parametrize("M,N,K,qt,bs,nested,bias,mt,splits", CONTRACT)
def test_weights_contract(M, N, K, qt, bs, nested, bias, mt, splits):
    p = make_problem(M, N, K, qt, bs, nested, bias, seed=2)
    assert_weights_contract(pair_call(p, mt, splits), p)


# identity activations: out[m, n] = 1 * W[n, m] + bias[n], one exact product per output -- the decoded weights
# themselves, bit for bit, for every (row, k) of the weight
@pytest.mark.parametrize("N,K,qt,bs,nested,mt", [
    (256, 320, "nf4", 64, True, 128), (130, 448, "fp4", 32, False, 64), (384, 1024, "nf4", 128, True, 32),
    (200, 512, "fp4", 256, False, 16), (128, 256, "nf4", 512, False, 128),
])
def test_decoded_weights_are_rna_tf32_of_dequantize_4bit(N, K, qt, bs, nested, mt):
    p = make_problem(K, N, K, qt, bs, nested, True, seed=10)
    p["x"] = torch.eye(K, device="cuda")
    got = pair_call(p, mt, 1)
    want = rna_tf32(p["W32"]).t() + p["bias"]  # one fp32 addition, as in the epilogue
    assert torch.equal(got.view(torch.int32), want.contiguous().view(torch.int32))


def test_the_tf32_instance_stops_at_128_tokens():
    p = make_problem(300, 256, 128, "nf4")
    out = torch.empty((300, 256), device="cuda")
    rc = nat.lib.cbnb_b200_gemm_4bit_pair(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), None, None, None, nat.ptr(out), None, 300, 256,
        128, 256, 64, nat.QT_ID["nf4"], 3, 256, 1, None, nat.stream())
    nat.check()
    assert rc == 100


@pytest.mark.parametrize("M,N,K,qt,bs,nested,bias", [
    (9, 4096, 4096, "nf4", 64, True, True),      # automatic tile and split
    (1000, 1000, 320, "fp4", 64, False, True),
    (4096, 512, 4096, "nf4", 64, False, False),
])
def test_weights_contract_through_the_dispatch(precision, M, N, K, qt, bs, nested, bias):
    p = make_problem(M, N, K, qt, bs, nested, bias, seed=3)
    assert nat.lib.cbnb_b200_gemm_4bit_path(M, N, K, bs, 3) == 1
    assert_weights_contract(native_call(p, 3), p)
    precision("tf32")
    assert torch.equal(op_call(p).view(torch.int32), native_call(p, 3).view(torch.int32))


def test_three_dimensional_input_through_the_op(precision):
    precision("tf32")
    p = make_problem(96, 384, 640, "nf4", 64, True, True, seed=4)
    x3 = p["x"].view(4, 24, 640)
    got = op_call(p, x3)
    torch.cuda.synchronize()
    assert got.shape == (4, 24, 384)
    assert_weights_contract(got, p, x3)


# ------------------------------------------------------------------------------------------------ 3. arbitrary fp32
@pytest.mark.parametrize("M,N,K,qt,bias", [(256, 1024, 4096, "nf4", False), (77, 300, 320, "fp4", True),
                                           (4096, 4096, 4096, "nf4", True)])
def test_arbitrary_fp32_activations_within_the_tf32_bound(precision, M, N, K, qt, bias):
    precision("tf32")
    p = make_problem(M, N, K, qt, 64, False, bias, seed=5, exact_acts=False)
    got = op_call(p)
    assert_tf32_bound(got, p["x"], p["W32"], p["bias"], "TF32 route")
    # the reference's route for fp32 from 8 tokens on: dequantise, then F.linear (cuBLAS, TF32 allowed)
    ref = torch.nn.functional.linear(p["x"], p["W32"], p["bias"])
    assert_tf32_bound(ref, p["x"], p["W32"], p["bias"], "dequantize + cuBLAS TF32")


# ------------------------------------------------------------------------------------------------ 4. determinism, routing
def test_split_k_is_deterministic():
    p = make_problem(16, 512, 4096, "nf4", 64, False, True, seed=6, exact_acts=False)
    outs = [native_call(p, 3) for _ in range(3)] + [pair_call(p, 16, 5) for _ in range(2)]
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    assert torch.equal(outs[1].view(torch.int32), outs[2].view(torch.int32))
    assert torch.equal(outs[3].view(torch.int32), outs[4].view(torch.int32))


def test_path_query_follows_the_threshold():
    path = nat.lib.cbnb_b200_gemm_4bit_path
    for M in (TF32_MIN_M, TF32_MIN_M + 1, 64, 4096):
        assert path(M, 4096, 4096, 64, 3) == 1
        assert path(M, 4096, 4096, 64, 0) == 2
    for M in range(1, TF32_MIN_M):
        assert path(M, 4096, 4096, 64, 3) == 2
    assert path(4096, 4096, 4000, 64, 3) == 2    # K % 64 != 0: the fp32 route
    assert path(4096, 4096, 4096, 48, 3) == 2    # blocksize not a power of two


def test_toggling_the_precision_switches_the_route(precision):
    p = make_problem(64, 384, 512, "nf4", 64, False, True, seed=7, exact_acts=False)
    precision("ieee")
    a = op_call(p)
    precision("tf32")
    b = op_call(p)
    precision("ieee")
    c = op_call(p)
    torch.cuda.synchronize()
    fp32, tf32 = native_call(p, 0), native_call(p, 3)
    assert torch.equal(a.view(torch.int32), fp32.view(torch.int32))
    assert torch.equal(c.view(torch.int32), fp32.view(torch.int32))
    assert torch.equal(b.view(torch.int32), tf32.view(torch.int32))
    assert not torch.equal(a, b), "the TF32 route gave the fp32 route's output"


# ------------------------------------------------------------------------------------------------ 5. layer, graphs
def test_linear4bit_fp32_under_tf32(precision):
    precision("tf32")
    K, N = 1024, 768
    g = torch.Generator(device="cpu").manual_seed(8)
    lin = torch.nn.Linear(K, N, bias=True)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(N, K, generator=g) / K**0.5)
        lin.bias.copy_(torch.randn(N, generator=g) * 0.1)
    layer = bnb.nn.Linear4bit(K, N, bias=True, compute_dtype=torch.float32, quant_type="nf4")
    layer.load_state_dict(lin.state_dict())
    layer = layer.cuda()
    x = torch.randn(2, 40, K, generator=g).cuda()
    with torch.no_grad():
        y = layer(x)
    W32 = bnb.functional.dequantize_4bit(layer.weight.data, layer.weight.quant_state).float()
    assert W32.dtype == torch.float32 and W32.shape == (N, K)
    assert_tf32_bound(y, x, W32, layer.bias.float(), "Linear4bit")


def test_cuda_graph_keeps_the_route_it_was_captured_with(precision):
    precision("tf32")
    p = make_problem(256, 1024, 1024, "nf4", 64, True, True, seed=9, exact_acts=False)
    static_x = p["x"].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        op_call(p, static_x)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_y = op_call(p, static_x)
    eager = op_call(p, static_x)
    precision("ieee")  # the replay keeps the route of the capture
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static_y.view(torch.int32), eager.view(torch.int32))
    static_x.copy_(torch.randn(256, 1024, device="cuda"))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static_y.view(torch.int32), native_call(p, 3, static_x).view(torch.int32))
