"""LLM.int8() with outlier columns inside CUDA graphs: the device-side outlier route.

* the compaction kernel gives the columns and count torch.nonzero gives;
* the route (compact -> prep with the count on the device -> GEMM reading the count) is bit-identical to the fused
  kernel of the eager route for 0 .. 64 outlier columns and zeroes the same codes; beyond 64 columns it is
  bit-identical to a CPU restatement of its fp32 sum and within the float64 bound of the eager tests;
* it runs with no host synchronisation;
* a captured Linear8bitLt(threshold=6.0) replays the eager forward for outlier sets that change between replays;
* the training forward under capture raises.
"""
import pytest
import torch

import bitsandbytes_b200 as bnb
from bitsandbytes_b200.backends import cuda as backend
from tests import _native as nat

pytestmark = pytest.mark.gpu

INV127 = 7.874015718698502e-3


def _ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    mant = 10 if dtype == torch.float16 else 7
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0**-24 if dtype == torch.float16 else 1e-38)))
    if dtype == torch.float16:
        e = e.clamp_min(-14)
    return torch.exp2(e - mant)


def _assert_within_fp64_bound(out, base, subA, subB, dtype, max_flip_rate=None):
    """out against base + subA . subBᵀ in float64 with the bound of the eager outlier tests: half an ulp of T plus fp32
    accumulation over J terms; optionally also a largest share of outputs off the float64 result rounded to T."""
    J = subA.shape[-1]
    o64 = subA.double() @ subB.double().t()
    exact64 = base.double() + o64
    diff = (out.double() - exact64).abs()
    tol = 0.5 * _ulp(exact64, dtype).double() * 1.001 + 2.0**-21 * (1 + o64.abs()) * J**0.5
    assert (diff <= tol).all(), f"{int((diff > tol).sum())} outputs off, worst excess {(diff - tol).max().item():.3e}"
    if max_flip_rate is not None:
        assert (out != exact64.to(dtype)).float().mean().item() < max_flip_rate


def _restated(base, subA, subB, dtype):
    """The route's arithmetic restated on the CPU: the outlier sum in fp32, one fma per column in column order (a
    product of two 16-bit floats is exact in float64, so rounding product + sum to float32 is the fma), added in fp32
    to the rounded int8 part `base` and rounded once to T."""
    a, b = subA.cpu().double(), subB.cpu().double()
    ol = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float32)
    for j in range(a.shape[1]):
        ol = (torch.outer(a[:, j], b[:, j]) + ol.double()).float()
    return (base.cpu().float() + ol).to(dtype)


def _bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ compaction
@pytest.mark.parametrize("K", [16, 80, 4096, 11008])
@pytest.mark.parametrize("pattern", ["none", "one", "ends", "all", "sparse", "dense"])
def test_outlier_compaction_equals_nonzero(K, pattern):
    g = torch.Generator().manual_seed(K)
    flags = torch.zeros(K, dtype=torch.int32)
    if pattern == "one":
        flags[int(torch.randint(K, (1,), generator=g))] = 1
    elif pattern == "ends":  # the first column and the last, which sits in a partial tile unless K % 1024 == 0
        flags[0] = flags[-1] = 1
    elif pattern == "all":
        flags[:] = 1
    elif pattern == "sparse":
        flags = (torch.rand(K, generator=g) < 0.03).to(torch.int32)
    elif pattern == "dense":
        flags = (torch.rand(K, generator=g) < 0.6).to(torch.int32)
    flags = flags.cuda()
    cols, count = backend.int8_outlier_compact(flags)
    torch.cuda.synchronize()
    nat.check()
    want = torch.nonzero(flags).view(-1)
    assert cols.dtype == torch.int32 and cols.shape == (K,)
    assert count.item() == want.numel()
    assert torch.equal(cols[: want.numel()].long(), want)


# ------------------------------------------------------------------------------------------------ the route
def _problem(M, N, K, J, dtype, with_bias, seed):
    """Random codes and statistics, activations whose columns `cols` hold large values, and the matching flags.  CA is
    NOT zeroed in the outlier columns: the route must do it."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    CA = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8).cuda()
    CB = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8).cuda()
    SCA = (torch.rand(M, generator=g) * 5 + 0.5).cuda()
    SCB = (torch.rand(N, generator=g) * 0.1 + 0.01).cuda()
    bias = torch.randn(N, generator=g).to(dtype).cuda() if with_bias else None
    A = (torch.randn(M, K, generator=g) * 2).to(dtype).cuda()
    cols = torch.randperm(K, generator=g)[:J].sort().values.cuda()
    A[:, cols] = (torch.randn(M, J, generator=g) * 4 + 9).to(dtype).cuda()
    flags = torch.zeros(K, dtype=torch.int32, device="cuda")
    flags[cols] = 1
    return CA, CB, SCA, SCB, bias, A, cols, flags


def _scaled_mm(CA, CB, SCA, SCB, bias, dtype):
    M, N, K = CA.shape[0], CB.shape[0], CA.shape[1]
    out = torch.full((M, N), float("nan"), device="cuda", dtype=dtype)
    rc = nat.lib.cbnb_b200_int8_scaled_mm(CA.data_ptr(), CB.data_ptr(), SCA.data_ptr(), SCB.data_ptr(), nat.ptr(bias),
                                          out.data_ptr(), M, N, K, 1 if dtype == torch.float16 else 2, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    return out


# the shapes and outlier counts of the fused-epilogue test of the eager route, plus no outlier column at all
@pytest.mark.parametrize("M,N,K,J", [(9, 24, 64, 1), (130, 300, 192, 5), (257, 1000, 1024, 8), (64, 512, 256, 9),
                                     (300, 384, 512, 41), (128, 256, 128, 64), (150, 200, 80, 24), (129, 260, 208, 32),
                                     (130, 300, 192, 0)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("with_bias", [False, True])
def test_route_is_bit_identical_to_the_fused_kernel(M, N, K, J, dtype, with_bias):
    CA, CB, SCA, SCB, bias, A, cols, flags = _problem(M, N, K, J, dtype, with_bias, seed=M * 7 + N + J)
    CA_route = CA.clone()
    out = backend.int8_mixed_mm_flags(A, CA_route, CB, SCA, SCB, flags, bias)
    torch.cuda.synchronize()
    nat.check()

    # the eager route: zero the outlier columns, build subA / subBT for exactly J columns, the JMAX-by-J kernel
    CA_eager = CA.clone()
    if J:
        backend.int8_zero_columns(CA_eager, cols)
    assert torch.equal(CA_route, CA_eager)
    if J == 0:
        want = _scaled_mm(CA_eager, CB, SCA, SCB, bias, dtype)
    else:
        did = 1 if dtype == torch.float16 else 2
        jpad = -(-J // 8) * 8
        subA = torch.empty((M, jpad), device="cuda", dtype=dtype)
        subBT = torch.empty((N, jpad), device="cuda", dtype=dtype)
        nat.lib.cbnb_b200_int8_outlier_prep(A.data_ptr(), CB.data_ptr(), SCB.data_ptr(), cols.data_ptr(), J, jpad, M, N,
                                            K, did, subA.data_ptr(), subBT.data_ptr(), nat.stream())
        want = torch.full((M, N), float("nan"), device="cuda", dtype=dtype)
        rc = nat.lib.cbnb_b200_int8_mixed_mm(CA_eager.data_ptr(), CB.data_ptr(), SCA.data_ptr(), SCB.data_ptr(),
                                             nat.ptr(bias), subA.data_ptr(), subBT.data_ptr(), jpad, want.data_ptr(), M,
                                             N, K, did, nat.stream())
        torch.cuda.synchronize()
        nat.check()
        assert rc == 0
    assert torch.equal(_bits(out), _bits(want)), f"{int((_bits(out) != _bits(want)).sum())} outputs differ"


@pytest.mark.parametrize("J", [65, 100, 300, 320])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("with_bias", [False, True])
def test_route_beyond_64_outlier_columns(J, dtype, with_bias):
    """Columns 64 .. J-1 are gathered from A and CB inside the GEMM, 64 at a time; J = 320 = K flags every column (and
    K ends half-way into a 128-byte k-block)."""
    M, N, K = 260, 300, 320
    CA, CB, SCA, SCB, bias, A, cols, flags = _problem(M, N, K, J, dtype, with_bias, seed=J)
    out = backend.int8_mixed_mm_flags(A, CA, CB, SCA, SCB, flags, bias)
    torch.cuda.synchronize()
    nat.check()
    assert (CA[:, cols] == 0).all()
    base = _scaled_mm(CA, CB, SCA, SCB, bias, dtype)  # the int8 part, from the codes the route zeroed
    subB = (CB[:, cols].float() * SCB.view(-1, 1) * INV127).to(dtype)
    assert torch.equal(_bits(out.cpu()), _bits(_restated(base, A[:, cols], subB, dtype)))
    _assert_within_fp64_bound(out, base, A[:, cols], subB, dtype, max_flip_rate=2e-3)


def test_route_does_not_synchronise():
    M, N, K = 300, 384, 512
    g = torch.Generator(device="cpu").manual_seed(5)
    A = (torch.randn(M, K, generator=g) * 2).clamp_(-5.5, 5.5).to(torch.float16).cuda()
    A[3, 17] = 40.0
    A[::5, 300] = -7.0
    CB = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8).cuda()
    SCB = (torch.rand(N, generator=g) * 0.1 + 0.01).cuda()
    bias = torch.randn(N, generator=g).to(torch.float16).cuda()

    def forward():
        CA, SCA, flags = backend.int8_vectorwise_quant_flags(A, 6.0)
        return backend.int8_mixed_mm_flags(A, CA, CB, SCA, SCB, flags, bias), flags

    want, flags = forward()  # (the first call of each kernel also sets its shared-memory limit)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with pytest.raises(RuntimeError):
            torch.nonzero(flags)  # the mode is active: the eager route's op would fail here
        got, _ = forward()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    nat.check()
    assert torch.equal(_bits(got), _bits(want))


# ------------------------------------------------------------------------------------------------ capture
def _layer(K, N, with_bias, has_fp16_weights, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    lin = torch.nn.Linear(K, N, bias=with_bias)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(N, K, generator=g) * 0.02)
        if with_bias:
            lin.bias.copy_(torch.randn(N, generator=g) * 0.1)
    layer = bnb.nn.Linear8bitLt(K, N, bias=with_bias, has_fp16_weights=has_fp16_weights, threshold=6.0)
    layer.load_state_dict(lin.state_dict())
    return layer.to("cuda").eval()


def _input(lead, K, J, dtype, seed):
    """Activations below the threshold except J columns, each of which crosses it in at least one token row."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(*lead, K, generator=g).clamp_(-5.5, 5.5)
    x2 = x.view(-1, K)
    cols = torch.randperm(K, generator=g)[:J].sort().values
    rows = torch.randint(x2.shape[0], (J,), generator=g)
    sign = torch.where(torch.rand(J, generator=g) < 0.5, -1.0, 1.0)
    x2[rows, cols] = (6.5 + 3 * torch.rand(J, generator=g)) * sign
    return x.to(dtype).cuda(), cols.cuda()


def _reference_parts(layer, x, cols, dtype):
    """The int8 part of the eager forward and the outlier operands, for the float64 bound."""
    K = x.shape[-1]
    x2 = x.reshape(-1, K)
    CA, SCA, _ = torch.ops.bitsandbytes.int8_vectorwise_quant.default(x2.to(torch.float16), 6.0)
    CA[:, cols] = 0
    CB, SCB = layer.state.CB, layer.state.SCB
    base = torch.ops.bitsandbytes.int8_scaled_mm.default(CA, CB, SCA, SCB, bias=layer.bias, dtype=dtype)
    subB = (CB[:, cols].float() * SCB.view(-1, 1) * INV127).to(dtype)
    return base, x2[:, cols], subB


@pytest.mark.parametrize("lead", [(1,), (16,), (300,), (1, 1), (4, 4), (2, 150)], ids=str)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("has_fp16_weights", [False, True])
@pytest.mark.parametrize("with_bias", [False, True])
def test_captured_linear8bitlt_replays_the_eager_forward(lead, dtype, has_fp16_weights, with_bias):
    K, N = 512, 328
    layer = _layer(K, N, with_bias, has_fp16_weights, seed=len(lead) * 1000 + lead[-1])
    static_x, _ = _input(lead, K, 41, dtype, seed=1)
    with torch.no_grad():
        # warm up on a side stream, as torch.cuda.graph asks: the weights are quantised there (fp16 master weights),
        # outside the capture
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            layer(static_x)
        torch.cuda.current_stream().wait_stream(side)
        idx_before = layer.state.idx
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_y = layer(static_x)
        assert layer.state.idx is idx_before  # the captured route leaves state.idx alone

        for J in (0, 5, 41, 100):
            x, cols = _input(lead, K, J, dtype, seed=10 + J)
            static_x.copy_(x)
            graph.replay()
            eager = layer(x)
            torch.cuda.synchronize()
            nat.check()
            got = static_y.clone()
            assert got.shape == (*lead, N) and got.dtype == dtype
            if J:
                assert torch.equal(layer.state.idx, cols)  # the input has exactly the outlier set intended
            if J <= 64:
                assert torch.equal(_bits(got), _bits(eager)), f"J={J}: {int((_bits(got) != _bits(eager)).sum())} differ"
            else:  # eager runs the reference's unfused chain here: both within the float64 bound, the replay exact
                base, subA, subB = _reference_parts(layer, x, cols, dtype)
                _assert_within_fp64_bound(got.reshape(-1, N), base, subA, subB, dtype)
                _assert_within_fp64_bound(eager.reshape(-1, N), base, subA, subB, dtype)
                assert torch.equal(_bits(got.reshape(-1, N).cpu()), _bits(_restated(base, subA, subB, dtype)))


def test_no_grad_forward_of_fp16_master_weights_takes_the_capture_route(monkeypatch):
    """Under no_grad the weight of has_fp16_weights=True still has requires_grad, and ctx.needs_input_grad reports it
    whatever the grad mode: the route must not mistake that for training."""
    layer = _layer(256, 200, True, True, seed=3)
    x, _ = _input((24,), 256, 9, torch.float16, seed=4)
    with torch.no_grad():
        eager = layer(x)
        assert layer.weight.requires_grad
        calls = []
        route = bnb.autograd._functions._int8_forward_captured
        monkeypatch.setattr(bnb.autograd._functions, "_int8_forward_captured", lambda *a: calls.append(1) or route(*a))
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
        got = layer(x)
    torch.cuda.synchronize()
    assert calls == [1]
    assert torch.equal(_bits(got), _bits(eager))


@pytest.mark.parametrize("has_fp16_weights,input_grad", [(True, False), (False, True)])
def test_training_forward_under_capture_raises(monkeypatch, has_fp16_weights, input_grad):
    layer = _layer(256, 200, True, has_fp16_weights, seed=5).train()
    x, _ = _input((24,), 256, 9, torch.float16, seed=6)
    x.requires_grad_(input_grad)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(RuntimeError, match="inference only"):
        layer(x)
