"""GPU: LLM.int8() training -- MatMul8bitLt.backward and Linear8bitLt(has_fp16_weights=True) -- against float64 / int64
restatements computed here from the inputs.

* grad_B, int8 part: the column codes and statistics of fp16(grad_out) and of fp16(A) (outlier columns zeroed), their
  exact int32 product, the pinned C restatement of the dequant epilogue: bit for bit, on the fused route (token count a
  multiple of 16) and on the zero-padded unfused one.  The outlier columns: g^T . A[:, idx] within half an fp16 ulp
  plus fp32 accumulation.
* grad_B against the true gradient g^T . A within a bound derived from the code step of both operands.
* grad_A against g . (CB * SCB / 127), grad_bias against g.sum(0), both within the accumulation bound of the dtype.
* the outlier fallback for more than 64 columns, and a short SGD run next to nn.Linear.
"""
from math import prod

import pytest
import torch

import bitsandbytes_b200 as bnb
from bitsandbytes_b200.autograd._functions import MatmulLtState
from tests import _native as nat
from tests.test_gpu_int8 import _reference_col_quant, expected_scaled_mm

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16, torch.float32]
UNIT = {torch.float16: 2.0**-11, torch.bfloat16: 2.0**-8, torch.float32: 2.0**-24}  # unit roundoff
# leading shape of A (2-D or 3-D), K, N: 128 tokens take the fused int8_scaled_mm for grad_B (its inner dimension is
# the token count), 40 tokens the unfused route with the token dimension zero-padded to 48
SHAPES = [((128,), 200, 136), ((40,), 200, 136), ((4, 32), 200, 136), ((5, 8), 200, 136), ((512,), 1024, 768)]
SHAPE_IDS = ["128", "40", "4x32", "5x8", "512-big"]


def _ulp16(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0**-24))).clamp_min(-14)
    return torch.exp2(e - 10)


@pytest.fixture
def native_calls(monkeypatch):
    """Records (name, args, return value) of the int8 GEMM entry points the library calls."""
    calls = []
    for name in ("cigemmlt_32", "cbnb_b200_int8_scaled_mm", "cbnb_b200_int8_mixed_mm", "cdequant_mm_int32_fp16"):
        def spy(*args, _fn=getattr(nat.lib, name), _name=name):
            rc = _fn(*args)
            calls.append((_name, args, rc))
            return rc
        monkeypatch.setattr(nat.lib, name, spy)
    return calls


def _problem(lead, K, N, dtype, threshold, with_bias, seed=0):
    """Activations whose token rows differ in scale, three outlier columns that also hold sub-threshold entries
    (threshold > 0), an incoming gradient whose token rows differ in scale, fp16 weights for fp16 inputs and fp32
    master weights otherwise."""
    g = torch.Generator(device="cpu").manual_seed(seed + prod(lead) * 7 + K + N + int(threshold))
    M = prod(lead)
    A = (torch.randn(M, K, generator=g) * 1.5 * torch.exp(torch.randn(M, 1, generator=g) * 0.4)).clamp_(-5.5, 5.5)
    if threshold > 0:
        cols = torch.randperm(K, generator=g)[:3]
        rows = torch.randperm(M, generator=g)[:max(2, M // 8)]
        sign = torch.where(torch.rand(len(rows), 3, generator=g) < 0.5, -1.0, 1.0)
        A[rows.view(-1, 1), cols] = sign * (6.5 + 3 * torch.rand(len(rows), 3, generator=g))
    G = torch.randn(M, N, generator=g) * torch.exp(torch.randn(M, 1, generator=g))
    W = torch.randn(N, K, generator=g) * 0.05
    bias = torch.randn(N, generator=g) * 0.1 if with_bias else None
    wdtype = torch.float16 if dtype == torch.float16 else torch.float32
    A = A.to(dtype).reshape(*lead, K).cuda().requires_grad_()
    B = W.to(wdtype).cuda().requires_grad_()
    bias = bias.to(dtype).cuda().requires_grad_() if with_bias else None
    return A, B, bias, G.to(dtype).reshape(*lead, N).cuda()


def _train_step(A, B, bias, G, threshold, calls=None):
    state = MatmulLtState()
    state.has_fp16_weights = True  # (class attributes, not constructor fields)
    state.threshold = threshold
    out = bnb.matmul(A, B, state=state, bias=bias)
    if calls is not None:
        calls.clear()  # record the backward's launches only
    out.backward(G)
    torch.cuda.synchronize()
    nat.check()
    return state


def _outlier_cols(A2h: torch.Tensor, threshold: float) -> torch.Tensor:
    if threshold <= 0:
        return torch.zeros(0, dtype=torch.int64, device=A2h.device)
    return (A2h.abs() >= threshold).any(dim=0).nonzero().view(-1)


def _assert_grad_B_route(calls, tokens):
    if tokens % 16 == 0:
        fused = [rc for name, args, rc in calls if name == "cbnb_b200_int8_scaled_mm" and args[8] == tokens]
        assert fused == [0], f"grad_B did not take the fused int8_scaled_mm: {[c[0] for c in calls]}"
    else:
        padded = -(-tokens // 16) * 16
        gemm = [(args[3], rc) for name, args, rc in calls if name == "cigemmlt_32"]
        assert gemm == [(tokens, 100), (padded, 0)], f"grad_B did not take the zero-padded GEMM: {gemm}"
        assert [name for name, _, _ in calls].count("cdequant_mm_int32_fp16") == 1


# ------------------------------------------------------------------------------------------ grad_B, int8 part
@pytest.mark.parametrize("lead,K,N", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("threshold", [0.0, 6.0])
@pytest.mark.parametrize("with_bias", [False, True])
def test_grad_B_int8_part_is_bit_exact(lead, K, N, dtype, threshold, with_bias, native_calls):
    A, B, bias, G = _problem(lead, K, N, dtype, threshold, with_bias)
    state = _train_step(A, B, bias, G, threshold, native_calls)
    _assert_grad_B_route(native_calls, prod(lead))

    A2 = A.detach().reshape(-1, K)
    G2 = G.reshape(-1, N)
    qg, sg = _reference_col_quant(G2.half(), 0.0)
    qa, sa = _reference_col_quant(A2.half(), threshold)
    idx = _outlier_cols(A2.half(), threshold)
    assert threshold == 0 or len(idx) == 3
    if threshold > 0:
        assert torch.equal(state.idx.sort().values, idx)
    qa[:, idx] = 0
    C = (qg.double().t() @ qa.double()).to(torch.int32)  # exact: |sum| <= tokens * 127^2, far below 2^53
    want = expected_scaled_mm(C, sg, sa, None, torch.float16).to(B.dtype)

    got = B.grad
    keep = torch.ones(K, dtype=torch.bool, device="cuda")
    keep[idx] = False
    bad = got[:, keep] != want[:, keep]
    assert not bad.any(), f"{int(bad.sum())} of {int(keep.sum()) * N} int8-part elements of grad_B differ"
    if len(idx):
        # the outlier columns: g^T . A[:, idx] of the operands in the input dtype, fp32 accumulation, one fp16 rounding
        exact = G2.double().t() @ A2[:, idx].double()
        acc = prod(lead) * 2.0**-24 * (G2.double().abs().t() @ A2[:, idx].double().abs())
        tol = 0.5 * _ulp16(exact.abs() + acc) + acc
        diff = (got[:, idx].double() - exact).abs()
        assert (diff <= tol).all(), f"{int((diff > tol).sum())} outlier-column elements off, " \
                                    f"worst excess {(diff - tol).max().item():.3e}"


# ------------------------------------------------------------------------------------------ grad_B, true gradient
@pytest.mark.parametrize("lead,K,N", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("threshold", [0.0, 6.0])
def test_grad_B_is_the_gradient_within_the_quantisation_bound(lead, K, N, dtype, threshold):
    A, B, bias, G = _problem(lead, K, N, dtype, threshold, False, seed=1)
    _train_step(A, B, bias, G, threshold)
    Ah = A.detach().reshape(-1, K).half()
    Gh = G.reshape(-1, N).half()
    exact = Gh.double().t() @ Ah.double()
    # per-element error of a dequantised code: half a code step (absmax / 254, widened for the fp32 division) plus the
    # fp16 rounding of a * 127 (2^-11 |a|); outlier entries carry no code step, their columns are exact up to the
    # cast of the operands to fp16, which the 2^-11 |a| term covers
    _, sa = _reference_col_quant(Ah, threshold)
    _, sg = _reference_col_quant(Gh, 0.0)
    ea = sa.double() / 254 * (1 + 2.0**-14) + 2.0**-11 * Ah.double().abs() + 2.0**-25
    eg = sg.double() / 254 * (1 + 2.0**-14) + 2.0**-11 * Gh.double().abs() + 2.0**-25
    mag = Gh.double().abs().t() @ Ah.double().abs()
    bound = Gh.double().abs().t() @ ea + eg.t() @ Ah.double().abs() + eg.t() @ ea
    bound += (prod(lead) * 2.0**-24 + 2.0**-20) * mag  # fp32 dequant arithmetic and outlier-term accumulation
    tol = bound + 0.5 * _ulp16(exact.abs() + bound)
    got = B.grad.double()
    diff = (got - exact).abs()
    rel = float((got - exact).norm() / exact.norm())
    assert (diff <= tol).all(), (f"grad_B is {rel:.3f} off the gradient (relative Frobenius); {int((diff > tol).sum())} "
                                 f"of {diff.numel()} elements outside the quantisation bound")


# ------------------------------------------------------------------------------------------ grad_A, grad_bias
def _check_grad_A(grad_A, G, CB, SCB, dtype):
    N = CB.shape[0]
    G2 = G.reshape(-1, N).double()
    W = CB.double() * SCB.double().view(-1, 1) / 127
    exact = (G2 @ W).view(grad_A.shape)
    mag = (G2.abs() @ W.abs()).view(grad_A.shape)
    # rounding of W to the dtype, of partial sums (reduced-precision reductions) and of the result; fp32 accumulation
    u = UNIT[dtype]
    tol = (3 * u + N * 2.0**-24 + 2.0**-22) * mag + 2.0**-25
    assert grad_A.dtype == dtype
    diff = (grad_A.double() - exact).abs()
    assert (diff <= tol).all(), f"grad_A: {int((diff > tol).sum())} elements off, worst excess {(diff - tol).max():.3e}"


def _check_grad_bias(grad_bias, G, dtype):
    N = G.shape[-1]
    G2 = G.reshape(-1, N).double()
    u = UNIT[dtype]
    tol = (2 * u + G2.shape[0] * 2.0**-24) * G2.abs().sum(0) + 2.0**-25
    assert grad_bias.shape == (N,) and grad_bias.dtype == dtype
    diff = (grad_bias.double() - G2.sum(0)).abs()
    assert (diff <= tol).all(), f"grad_bias: {int((diff > tol).sum())} elements off"


@pytest.mark.parametrize("lead", [(128,), (40,), (4, 32), (5, 8)], ids=["128", "40", "4x32", "5x8"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("threshold", [0.0, 6.0])
@pytest.mark.parametrize("with_bias", [False, True])
def test_grad_A_and_grad_bias_with_fp16_weights(lead, dtype, threshold, with_bias):
    K, N = 200, 136
    A, B, bias, G = _problem(lead, K, N, dtype, threshold, with_bias, seed=2)
    state = _train_step(A, B, bias, G, threshold)
    # the weight codes the backward dequantises, against a float64 restatement of the row quantisation (exact
    # statistics; codes within one step where w * 127 / absmax sits on a rounding boundary)
    Bh = B.detach().half().double()
    rowmax = Bh.abs().amax(dim=1)
    assert torch.equal(state.SCB.double(), rowmax)
    assert (state.CB.double() - torch.round(Bh * 127 / rowmax.view(-1, 1))).abs().max() <= 1
    _check_grad_A(A.grad, G, state.CB, state.SCB, dtype)
    if with_bias:
        _check_grad_bias(bias.grad, G, dtype)


@pytest.mark.parametrize("lead", [(128,), (5, 8)], ids=["128", "5x8"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("threshold", [0.0, 6.0])
@pytest.mark.parametrize("with_bias", [False, True])
def test_grad_A_with_int8_weights(lead, dtype, threshold, with_bias):
    K, N = 200, 136
    A, B, bias, G = _problem(lead, K, N, dtype, threshold, with_bias, seed=3)
    layer = bnb.nn.Linear8bitLt(K, N, bias=with_bias, has_fp16_weights=False, threshold=threshold)
    with torch.no_grad():
        layer.weight.copy_(B.detach().float().cpu())
        if with_bias:
            layer.bias.copy_(bias.detach().float().cpu())
    layer = layer.cuda()
    out = layer(A)
    out.backward(G)
    torch.cuda.synchronize()
    nat.check()
    assert layer.weight.dtype == torch.int8 and layer.weight.grad is None
    _check_grad_A(A.grad, G, layer.state.CB, layer.state.SCB, dtype)
    if with_bias:
        _check_grad_bias(layer.bias.grad, G, dtype)


# ------------------------------------------------------------------------------------------ > 64 outlier columns
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("with_bias", [False, True])
def test_mixed_scaled_mm_with_more_than_64_outlier_columns(dtype, with_bias, native_calls):
    """The fused kernel holds at most 64 outlier columns; beyond that the op runs int8_scaled_mm and adds the outlier
    term with addmm.  Against the int8 part from the exact accumulators plus a float64 outlier product."""
    M, N, K, J = 96, 200, 256, 70
    g = torch.Generator(device="cpu").manual_seed(J + M)
    CA = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8).cuda()
    CB = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8).cuda()
    SCA = (torch.rand(M, generator=g) * 5 + 0.5).cuda()
    SCB = (torch.rand(N, generator=g) * 0.1 + 0.01).cuda()
    bias = torch.randn(N, generator=g).to(dtype).cuda() if with_bias else None
    A = (torch.randn(M, K, generator=g) * 2).to(dtype).cuda()
    cols = torch.randperm(K, generator=g)[:J].sort().values.cuda()
    A[:, cols] = (torch.randn(M, J, generator=g) * 4 + 9).to(dtype).cuda()
    CA[:, cols] = 0
    out, subA = torch.ops.bitsandbytes.int8_mixed_scaled_mm(A, CA, CB, SCA, SCB, cols, bias)
    torch.cuda.synchronize()
    nat.check()
    names = [name for name, _, _ in native_calls]
    assert "cbnb_b200_int8_mixed_mm" not in names and "cbnb_b200_int8_scaled_mm" in names
    assert torch.equal(subA, A[:, cols])

    C = (CA.double() @ CB.double().t()).to(torch.int32)
    base = expected_scaled_mm(C, SCA, SCB, bias, dtype).double()
    subB = (CB[:, cols].float() * SCB.view(-1, 1) * (1.0 / 127.0)).to(dtype).double()  # reference formula
    o64 = A[:, cols].double() @ subB.t()
    exact = base + o64
    mag = A[:, cols].double().abs() @ subB.abs().t()
    # one rounding to the dtype, fp32 accumulation, and room for one more rounding of the product (reduced-precision
    # reductions)
    u = UNIT[dtype]
    tol = u * (exact.abs() + mag) * 1.001 + u * mag + J * 2.0**-24 * mag
    diff = (out.double() - exact).abs()
    assert (diff <= tol).all(), f"{int((diff > tol).sum())} outputs off, worst excess {(diff - tol).max().item():.3e}"


# ------------------------------------------------------------------------------------------ training
@pytest.mark.parametrize("threshold", [0.0, 6.0])
def test_linear8bitlt_training_tracks_nn_linear(threshold):
    """20 SGD steps of Linear8bitLt(has_fp16_weights=True) and nn.Linear from the same weights on the same fp16
    batches: the int8 run must end near the fp32 one, relative to how far the fp32 one moved, and lower the loss."""
    K, N, M, steps = 256, 192, 64, 20
    g = torch.Generator(device="cpu").manual_seed(7)
    W0 = torch.randn(N, K, generator=g) * 0.05
    b0 = torch.randn(N, generator=g) * 0.1
    teacher = torch.randn(N, K, generator=g) * 0.08
    batches = []
    for _ in range(steps):
        x = (torch.randn(M, K, generator=g) * 1.5).clamp_(-5.5, 5.5)
        if threshold > 0:
            x[::5, 17] = 7.5
            x[1::9, 130] = -8.0
        batches.append((x.half().cuda(), (x @ teacher.t()).cuda()))

    lin = torch.nn.Linear(K, N).cuda()
    layer = bnb.nn.Linear8bitLt(K, N, has_fp16_weights=True, threshold=threshold)
    with torch.no_grad():
        lin.weight.copy_(W0)
        lin.bias.copy_(b0)
        layer.weight.copy_(W0)
        layer.bias.copy_(b0)
    layer = layer.cuda()

    def run(model, cast):
        opt = torch.optim.SGD(model.parameters(), lr=4.0)
        path, losses = [model.weight.detach().float().clone()], []
        for x, y in batches:
            opt.zero_grad()
            loss = torch.nn.functional.mse_loss(model(cast(x)).float(), y)
            loss.backward()
            opt.step()
            losses.append(loss.item())
            path.append(model.weight.detach().float().clone())
        return path, losses

    want, want_losses = run(lin, lambda x: x.float())
    got, losses = run(layer, lambda x: x)
    torch.cuda.synchronize()
    nat.check()
    moved = float((want[-1] - want[0]).norm())
    off = float((got[-1] - want[-1]).norm())
    assert off < 0.05 * moved, f"end point {off:.3e} away from nn.Linear's after a path of {moved:.3e}"
    assert losses[-1] < 0.5 * losses[0], f"loss {losses[0]:.4f} -> {losses[-1]:.4f}"
