"""GPU tests of the public Python surface (functional / autograd / nn / parallel): the call a
user of the reference would make, on the sm_90a kernels.  Tolerances are the reference's own
test bounds (cited per test)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bnb():
    import bitsandbytes_b200 as bnb

    return bnb


@pytest.mark.parametrize("quant_type", ["nf4", "fp4"])
@pytest.mark.parametrize("blocksize", [64, 128, 4096])
@pytest.mark.parametrize("nested", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_quantize_dequantize_4bit_error_tables(bnb, quant_type, blocksize, nested, dtype):
    """Round-trip mean |err| on N(0,1) inside the reference's per-blocksize table
    (reference tests/test_functional.py:606-651, measured on an RTX 4090, mean + 7 sigma)."""
    F = bnb.functional
    A = torch.randn(1024, 1024, device="cuda", dtype=dtype)
    q, qs = F.quantize_4bit(A, blocksize=blocksize, quant_type=quant_type, compress_statistics=nested)
    assert q.dtype == torch.uint8 and q.shape == (1024 * 1024 // 2, 1)
    assert qs.nested == nested and qs.shape == A.shape and qs.dtype == dtype
    D = F.dequantize_4bit(q, qs)
    assert D.dtype == dtype and D.shape == A.shape
    err = (A.float() - D.float()).abs().mean().item()
    # (mean, std) from the reference's table; threshold = mean + 7 sigma as in the reference
    table = {("nf4", 64): (0.072798, 0.000074), ("nf4", 128): (0.076831, 0.000091), ("nf4", 4096): (0.092547, 0.000360),
             ("fp4", 64): (0.096543, 0.000111), ("fp4", 128): (0.102969, 0.000134), ("fp4", 4096): (0.129536, 0.000612)}
    mean, std = table[(quant_type, blocksize)]
    bound = mean + 7 * std
    assert err < bound * (1.01 if nested else 1.0), err


@pytest.mark.parametrize("storage", [torch.uint8, torch.bfloat16, torch.float16, torch.float32])
def test_quant_storage_views_hold_the_same_bytes(bnb, storage):
    F = bnb.functional
    A = torch.randn(256, 128, device="cuda", dtype=torch.bfloat16)
    q8, s8 = F.quantize_4bit(A, quant_type="nf4", quant_storage=torch.uint8)
    q, s = F.quantize_4bit(A, quant_type="nf4", quant_storage=storage)
    assert q.dtype == storage and torch.equal(q.view(torch.uint8).reshape(-1), q8.reshape(-1))
    assert torch.equal(F.dequantize_4bit(q, s), F.dequantize_4bit(q8, s8))
    x = torch.randn(5, 128, device="cuda", dtype=torch.bfloat16)
    assert torch.equal(bnb.matmul_4bit(x, q.t(), s), bnb.matmul_4bit(x, q8.t(), s8))


def test_blockwise_8bit_api_round_trip_and_nested(bnb):
    F = bnb.functional
    A = torch.randn(1024, 1024, device="cuda")
    q, st = F.quantize_blockwise(A)
    D = F.dequantize_blockwise(q, st)
    err = (A - D).abs()
    assert err.mean().item() < 0.011 and (err / (A.abs() + 1e-8)).mean().item() < 0.018  # reference :113-169
    q2, st2 = F.quantize_blockwise(A, nested=True)
    assert st2.nested and torch.equal(q, q2)
    D2 = F.dequantize_blockwise(q2, st2)
    assert (D - D2).abs().max().item() < 0.05
    out = torch.empty_like(A)
    assert F.dequantize_blockwise(q, st, out=out) is out and torch.equal(out, D)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("nested", [False, True])
@pytest.mark.parametrize("M", [1, 7, 96, 300])
def test_matmul_4bit_equals_dequantize_then_matmul(bnb, dtype, nested, M):
    """matmul_4bit == x @ dequantize_4bit(W)^T in fp32 up to one rounding (reference
    tests/test_functional.py:989-1013 allows mean |err| < 0.115 vs the unquantised product)."""
    F = bnb.functional
    N, K = 1024, 512
    W = (torch.randn(N, K, device="cuda") / K**0.5).to(dtype)
    x = torch.randn(M, K, device="cuda", dtype=dtype)
    bias = torch.randn(N, device="cuda", dtype=dtype)
    qW, qs = F.quantize_4bit(W, quant_type="nf4", compress_statistics=nested)
    y = bnb.matmul_4bit(x, qW.t(), qs, bias=bias)
    ref = x.float() @ F.dequantize_4bit(qW, qs).float().t() + bias.float()
    assert y.dtype == dtype and y.shape == (M, N)
    eps = {torch.bfloat16: 2.0**-8, torch.float16: 2.0**-11, torch.float32: 2.0**-20}[dtype]
    assert ((y.float() - ref).abs() <= eps * 1.01 * ref.abs() + 1e-4).all()
    full = x.float() @ W.float().t() + bias.float()
    assert (y.float() - full).abs().mean().item() < 0.115


def test_matmul_4bit_legacy_kn_orientation_warns(bnb):
    F = bnb.functional
    Wt = torch.randn(128, 256, device="cuda", dtype=torch.bfloat16)  # [K, N]
    q, qs = F.quantize_4bit(Wt, quant_type="nf4")
    x = torch.randn(4, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.warns(DeprecationWarning):
        y = bnb.matmul_4bit(x, q, qs)
    assert y.shape == (4, 256)


@pytest.mark.parametrize("quant_type", ["nf4", "fp4"])
@pytest.mark.parametrize("compress", [False, True])
def test_linear4bit_module(bnb, quant_type, compress):
    lin = torch.nn.Linear(512, 384, bias=True)
    m = bnb.nn.Linear4bit(512, 384, bias=True, compute_dtype=torch.bfloat16, quant_type=quant_type,
                          compress_statistics=compress)
    m.load_state_dict(lin.state_dict())
    m = m.to("cuda")
    assert m.weight.dtype == torch.uint8 and m.weight.bnb_quantized and m.weight.quant_state.nested == compress
    assert m.quant_state is m.weight.quant_state
    x = torch.randn(3, 17, 512, device="cuda", dtype=torch.float16)
    y = m(x)
    assert y.dtype == torch.float16 and y.shape == (3, 17, 384)
    ref = torch.nn.functional.linear(x.float(), lin.weight.cuda().float(), lin.bias.cuda().float())
    assert (y.float() - ref).abs().mean().item() < (0.045 if quant_type == "nf4" else 0.06)
    # state dict round trip through from_prequantized
    sd = m.state_dict()
    stats = {k[len("weight."):]: v for k, v in sd.items() if k.startswith("weight.")}
    m2 = bnb.nn.Linear4bit(512, 384, bias=True, compute_dtype=torch.bfloat16, quant_type=quant_type,
                           compress_statistics=compress)
    m2.weight = bnb.nn.Params4bit.from_prequantized(sd["weight"], stats, device="cuda", module=m2)
    m2.bias = torch.nn.Parameter(sd["bias"].clone())
    assert torch.equal(m2.cuda()(x), y)


def test_matmul_4bit_backward_matches_dequantized_weight(bnb):
    """grad_A = grad_out @ dequantize_4bit(W) (reference autograd/_functions.py:364-386)."""
    F = bnb.functional
    W = (torch.randn(256, 128, device="cuda") / 11).to(torch.bfloat16)
    qW, qs = F.quantize_4bit(W, quant_type="nf4")
    x = torch.randn(9, 128, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    bias = torch.randn(256, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    y = bnb.matmul_4bit(x, qW.t(), qs, bias=bias)
    g = torch.randn_like(y)
    y.backward(g)
    Wd = F.dequantize_4bit(qW, qs)
    assert torch.allclose(x.grad.float(), (g.float() @ Wd.float()), atol=2e-2, rtol=2e-2)
    assert torch.allclose(bias.grad.float(), g.float().sum(0), atol=5e-2, rtol=2e-2)


@pytest.mark.parametrize("threshold", [0.0, 6.0])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_linear8bitlt_module(bnb, threshold, dtype):
    """reference tests/test_modules.py:65-130 / test_autograd.py:36-140: <= ~2% of elements outside
    atol 0.01 / rtol 0.1 of the fp16 linear."""
    lin = torch.nn.Linear(1024, 768, bias=True)
    m = bnb.nn.Linear8bitLt(1024, 768, bias=True, has_fp16_weights=False, threshold=threshold)
    m.load_state_dict(lin.state_dict())
    m = m.to("cuda").eval()
    assert m.weight.dtype == torch.int8 and m.weight.SCB is not None
    x = torch.randn(64, 1024, device="cuda", dtype=dtype)
    if threshold > 0:
        x[:, [3, 500, 801]] = 9.0
    y = m(x)
    assert y.dtype == dtype and y.shape == (64, 768)
    assert m.state.CB is not None and m.weight.CB is None  # moved into the state on first forward
    ref = torch.nn.functional.linear(x.float(), lin.weight.cuda().float(), lin.bias.cuda().float())
    close = torch.isclose(y.float(), ref, atol=0.03 if threshold == 0 else 0.05, rtol=0.1)
    assert (~close).float().mean().item() < 0.03
    if threshold > 0:
        assert sorted(m.state.idx.tolist()) == [3, 500, 801]
    sd = m.state_dict()
    assert "SCB" in sd and sd["weight"].dtype == torch.int8


def test_int8_ops_through_dispatcher(bnb):
    F = bnb.functional
    A = torch.randn(33, 256, device="cuda", dtype=torch.float16)
    A[:, 7] = -8
    q, stats, cols = F.int8_vectorwise_quant(A, threshold=6.0)
    assert cols.tolist() == [7] and (q[:, 7] == 0).all()
    masked = A.float().abs()
    masked[:, 7] = 0
    assert torch.equal(stats, masked.amax(1))
    q0, stats0, cols0 = F.int8_vectorwise_quant(A)
    assert cols0 is None and torch.equal(stats0, A.float().abs().amax(1))
    W = torch.randint(-127, 128, (48, 256), dtype=torch.int8, device="cuda")
    C = F.int8_linear_matmul(q0, W)
    assert torch.equal(C, (q0.double() @ W.double().t()).to(torch.int32))
    out = F.int8_mm_dequant(C, stats0, torch.rand(48, device="cuda") + 0.5)
    assert out.dtype == torch.float16 and out.shape == (33, 48)
    deq = F.int8_vectorwise_dequant(q0, stats0)
    assert (deq - A.float()).abs().max().item() < stats0.max().item() / 127 * 0.51 + 1e-3
    r, c, rs, cs, oc = F.int8_double_quant(A, threshold=6.0)
    assert torch.equal(r, q) and c.shape == A.shape and oc.tolist() == [7]


def test_opcheck_on_the_hot_ops(bnb):
    F = bnb.functional
    A = torch.randn(8, 128, device="cuda", dtype=torch.bfloat16)
    W = torch.randn(64, 128, device="cuda", dtype=torch.bfloat16)
    qW, qs = F.quantize_4bit(W, quant_type="nf4")
    torch.library.opcheck(torch.ops.bitsandbytes.gemm_4bit.default, (A, qW, [64, 128], qs.absmax, 64, "nf4"))
    torch.library.opcheck(torch.ops.bitsandbytes.quantize_4bit.default, (W, 64, "nf4", torch.uint8))
    torch.library.opcheck(torch.ops.bitsandbytes.dequantize_4bit.default, (qW, qs.absmax, 64, "nf4", [64, 128], torch.bfloat16))
    code = F.create_dynamic_map().cuda()
    torch.library.opcheck(torch.ops.bitsandbytes.quantize_blockwise.default, (torch.randn(4096, device="cuda"), code, 256))


@pytest.mark.parametrize("nested", [False, True])
def test_column_shards_reproduce_the_single_gpu_result(bnb, nested):
    """C4 shape family on one GPU: the 8 row-shards of a globally quantised FP4 weight, each run
    through the fused kernel into its columns of the full output, equal the unsharded GEMM bit
    for bit (SURVEY.md section 8e: quantise once globally, then slice)."""
    from bitsandbytes_b200.parallel import ColumnParallelLinear4bit, slice_quantized_weight

    F = bnb.functional
    N, K, M = 3584, 1024, 48
    W = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    qW, qs = F.quantize_4bit(W, quant_type="fp4", compress_statistics=nested)
    full = bnb.matmul_4bit(x, qW.t(), qs)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    world = 7 if not nested else 2   # nested needs rows*K/64 % 256 == 0
    for r in range(world):
        layer = ColumnParallelLinear4bit(slice_quantized_weight(qW, qs, world, r), N)
        s = layer.shard
        layer.local_forward(x, out[:, s.row0:s.row0 + s.rows], N)
    torch.cuda.synchronize()
    assert torch.equal(out, full)
