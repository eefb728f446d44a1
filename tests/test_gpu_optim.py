"""GPU parity of the optimizer updates (SURVEY.md section 8 row f-4), through the C ABI:

* every optimizer x dtype x {32-bit, blockwise 8-bit state} against the numpy restatement (oracle/optim_ref.py:
  exact division / sqrt, so within a few ulp; the 8-bit codes may differ only next to a code-book midpoint);
* the same inputs through the reference CUDA library built from the reference sources (strict: same symbols,
  same arguments, legacy default stream);
* the public classes (bnb.optim.*) against torch.optim on a small model, state-dict round trip, paged state.
"""
import numpy as np
import pytest
import torch

from oracle import optim_ref as R
from tests import _native as nat

pytestmark = pytest.mark.gpu

OPT_ID = {"adam": 0, "momentum": 1, "rmsprop": 2, "adagrad": 3, "lion": 4, "ademamix": 5}
HYPER = {  # lr, beta1, beta2, beta3, alpha, eps, weight_decay
    "adam": (1e-3, 0.9, 0.999, 0.0, 0.0, 1e-8, 0.01),
    "momentum": (1e-2, 0.9, 0.0, 0.0, 0.0, 0.0, 0.01),
    "rmsprop": (1e-2, 0.99, 0.0, 0.0, 0.0, 1e-8, 0.01),
    "adagrad": (1e-2, 0.0, 0.0, 0.0, 0.0, 1e-10, 0.01),
    "lion": (1e-4, 0.9, 0.99, 0.0, 0.0, 0.0, 0.01),
    "ademamix": (1e-3, 0.9, 0.999, 0.9999, 5.0, 1e-8, 0.01),
}
ULP = {"fp32": 2.0**-23, "fp16": 2.0**-10, "bf16": 2.0**-7}


def _f32(t):
    return t.detach().float().cpu().numpy()


def _codes():
    import bitsandbytes_b200.functional as F

    return F.create_dynamic_map(signed=True).cuda().contiguous(), F.create_dynamic_map(signed=False).cuda().contiguous()


def _inputs(n, dtype, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    p = (torch.randn(n, generator=g) * 0.5).to(nat.DTYPE[dtype]).cuda()
    grad = (torch.randn(n, generator=g) * 0.1).to(nat.DTYPE[dtype]).cuda()
    return p, grad


def _close(got, want, dtype, what, ulps=2.0, atol=1e-7, scale_ulps=0.0):
    """|got - want| <= ulps * ulp(want) + atol + scale_ulps * ulp(max |want|): the last term covers sums whose terms are
    larger than the result (an fma contracted differently moves the result by an ulp of the TERMS)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    ok = np.isfinite(want)
    assert (np.isfinite(got) == ok).all(), f"{what}: non-finite values differ"
    scale = np.abs(want[ok]).max() if ok.any() else 0.0
    tol = ulps * ULP[dtype] * np.abs(want) + atol + scale_ulps * ULP[dtype] * scale
    bad = ok & (np.abs(got - want) > tol)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} off, worst {np.abs(got - want)[ok].max():.3e}"


@pytest.mark.parametrize("name", list(OPT_ID))
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("n", [4096, 1000])
def test_32bit_update_matches_the_oracle(name, dtype, n):
    lr, b1, b2, b3, alpha, eps, wd = HYPER[name]
    p, grad = _inputs(n, dtype, 7 + n)
    two = name in ("adam", "ademamix")
    s1 = torch.zeros((2, n) if name == "ademamix" else (n,), device="cuda")
    s2 = torch.zeros(n, device="cuda") if two else None
    for step in (1, 2, 3):
        grad = (grad.float() * 0.9 + 0.01).to(grad.dtype)
        want = R.update_32bit(name, dtype, _f32(grad), _f32(p), _f32(s1), None if s2 is None else _f32(s2), step, lr, b1, b2,
                              b3, alpha, eps, wd)
        rc = nat.lib.cbnb_b200_optimizer_update_32bit(OPT_ID[name], nat.DTYPE_ID[dtype], nat.ptr(grad), nat.ptr(p),
                                                      nat.ptr(s1), nat.ptr(s2), None, 0.0, 0.0, b1, b2, b3, alpha, eps, wd,
                                                      step, lr, 1.0, False, n, nat.stream())
        torch.cuda.synchronize()
        nat.check()
        assert rc == 0
        _close(_f32(p), want[0], dtype, f"{name} {dtype} step {step}: p", ulps=1.01)
        _close(_f32(s1), want[1], "fp32", f"{name} step {step}: state1", ulps=8, atol=1e-9)
        if two:
            _close(_f32(s2), want[2], "fp32", f"{name} step {step}: state2", ulps=8, atol=1e-12)


@pytest.mark.parametrize("name", ["adam", "momentum", "rmsprop", "adagrad"])
def test_32bit_trust_ratio_matches_the_oracle(name):
    """max_unorm > 0 (LAMB / LARS): the squared update norm is accumulated first and clips the step."""
    lr, b1, b2, b3, alpha, eps, wd = HYPER[name]
    n, dtype = 5000, "fp32"
    p, grad = _inputs(n, dtype, 3)
    s1 = torch.rand(n, device="cuda") * 0.01
    s2 = torch.rand(n, device="cuda") * 0.001 if name == "adam" else None
    unorm = torch.zeros(1, device="cuda")
    max_unorm = 0.01
    pn = float(torch.norm(p.float()))
    want = R.update_32bit("lamb" if name == "adam" else name, dtype, _f32(grad), _f32(p), _f32(s1),
                          None if s2 is None else _f32(s2), 2, lr, b1, b2, b3, alpha, eps, 0.0, max_unorm=max_unorm)
    nat.lib.cbnb_b200_optimizer_update_32bit(OPT_ID[name], 0, nat.ptr(grad), nat.ptr(p), nat.ptr(s1), nat.ptr(s2),
                                             nat.ptr(unorm), max_unorm, pn, b1, b2, b3, alpha, eps, 0.0, 2, lr, 1.0, False, n,
                                             nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert abs(float(unorm) - float(want[3])) <= 1e-4 * abs(float(want[3]))
    _close(_f32(p), want[0], dtype, f"{name} trust ratio: p", ulps=64)


def _blockwise_state(name, n, seed):
    """A plausible mid-training 8-bit state: random codes and per-block absmax."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    nb = -(-n // 256)
    two = name in ("adam", "ademamix")
    rows = 2 if name == "ademamix" else 1
    lo = 128 if name in ("rmsprop", "adagrad") else 0  # a second-moment state is never negative
    c1 = torch.randint(lo, 256, (rows, n) if rows == 2 else (n,), generator=g, dtype=torch.uint8).cuda()
    c2 = torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8).cuda() if two else None
    a1 = (torch.rand(rows * nb, generator=g) * 0.05 + 1e-3).cuda()
    a2 = (torch.rand(nb, generator=g) * 0.002 + 1e-5).cuda() if two else None
    return c1, c2, a1, a2


@pytest.mark.parametrize("name", list(OPT_ID))
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("n", [4096, 1000, 256 * 37])
def test_8bit_blockwise_update_matches_the_oracle(name, dtype, n):
    if name == "ademamix" and n % 256:
        pytest.skip("the reference indexes the slow EMA's absmax at (n + i) / 256: defined for n % 256 == 0 only")
    lr, b1, b2, b3, alpha, eps, wd = HYPER[name]
    p, grad = _inputs(n, dtype, 11 + n)
    code1, code2 = _codes()
    c1, c2, a1, a2 = _blockwise_state(name, n, 5 + n)
    two = c2 is not None
    for step in (1, 2, 5):
        p_before = _f32(p)
        want = R.update_8bit_blockwise(name, dtype, _f32(grad), _f32(p), c1.cpu().numpy(), None if c2 is None else c2.cpu().numpy(),
                                       code1.cpu().numpy(), code2.cpu().numpy(), _f32(a1), None if a2 is None else _f32(a2),
                                       step, lr, b1, b2, b3, alpha, eps, wd)
        rc = nat.lib.cbnb_b200_optimizer_update_8bit_blockwise(
            OPT_ID[name], nat.DTYPE_ID[dtype], nat.ptr(p), nat.ptr(grad), nat.ptr(c1), nat.ptr(c2), b1, b2, b3, alpha, eps, step,
            lr, nat.ptr(code1), nat.ptr(code2) if two else None, nat.ptr(a1), nat.ptr(a2), wd, 1.0, False, n, nat.stream())
        torch.cuda.synchronize()
        nat.check()
        assert rc == 0
        np.testing.assert_allclose(_f32(a1), want[3], rtol=2e-6, atol=1e-12, err_msg=f"{name} absmax1")
        if two:
            np.testing.assert_allclose(_f32(a2), want[4], rtol=2e-6, atol=1e-20, err_msg=f"{name} absmax2")
        # the parameter: the reference's (and our) __powf / div.approx / sqrt.approx move the UPDATE by up to ~1e-3 of
        # itself (1 - __powf(beta2, step) cancels), the oracle computes them exactly
        upd = np.abs(want[0] - p_before)
        _close(_f32(p), want[0], dtype, f"{name} {dtype} step {step}: p", ulps=1.01, atol=2e-3 * float(upd[np.isfinite(upd)].max()))
        same1 = (c1.cpu().numpy() == want[1]).mean()
        assert same1 > 0.995, f"{name}: state1 codes agree only at {same1:.4f}"
        d1 = np.abs(c1.cpu().numpy().astype(np.int64) - want[1].astype(np.int64))
        assert d1.max() <= 1, f"{name}: a state1 code is {d1.max()} entries away from the oracle's"
        if two:
            same2 = (c2.cpu().numpy() == want[2]).mean()
            assert same2 > 0.995, f"{name}: state2 codes agree only at {same2:.4f}"
        grad = (grad.float() * 0.7 - 0.02).to(grad.dtype)


def _ref_name32(name, dtype):
    if name in ("adam", "lion", "ademamix"):
        return f"c{name}32bit_grad_{dtype}"
    return None if dtype == "bf16" else f"c{name}32bit_grad_{'32' if dtype == 'fp32' else '16'}"


@pytest.mark.parametrize("name", list(OPT_ID))
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
def test_32bit_update_equals_the_reference_cuda_library(name, dtype):
    sym = _ref_name32(name, dtype)
    ref = nat.ref_cuda()
    # The reference exports no bf16 variant of momentum / RMSprop / Adagrad.  Its 32-bit kernels are one template
    # over the parameter type that rounds to T only the gradient after weight decay and the stored parameter, so
    # without weight decay its fp32 variant run on the bf16 values, with the parameters rounded to bf16 after every
    # step, is what a bf16 variant computes.  (Weight decay: the fp32 / fp16 comparisons here and the oracle tests.)
    emulate = sym is None
    ours_sym = sym if not emulate else f"cbnb_b200_optimizer_update_32bit[{name}, bf16]"
    fn_ref = getattr(ref, _ref_name32(name, "fp32") if emulate else sym)
    if emulate:  # our bf16 variant through the native entry (the reference ABI has no name for it)
        def fn_ours(*args):
            assert nat.lib.cbnb_b200_optimizer_update_32bit(OPT_ID[name], nat.DTYPE_ID["bf16"], *args, nat.stream()) == 0
    else:
        fn_ours = getattr(nat.lib, sym)
    lr, b1, b2, b3, alpha, eps, wd = HYPER[name]
    if emulate:
        wd = 0.0
    n = 70001
    two = name in ("adam", "ademamix")
    out = []
    for fn in (fn_ref, fn_ours):
        p, grad = _inputs(n, dtype, 21)
        widen = emulate and fn is fn_ref
        if widen:
            p = p.float()
        s1 = torch.zeros((2, n) if name == "ademamix" else (n,), device="cuda")
        s2 = torch.zeros(n, device="cuda") if two else None
        for step in (1, 2, 3, 4):
            g_in = grad.float() if widen else grad
            torch.cuda.synchronize()
            fn(nat.ptr(g_in), nat.ptr(p), nat.ptr(s1), nat.ptr(s2), None, 0.0, 0.0, b1, b2, b3, alpha, eps, wd, step, lr, 1.0,
               False, n)
            torch.cuda.synchronize()
            if widen:
                p.copy_(p.to(torch.bfloat16).float())
            grad = (grad.float() * 0.9 + 0.01).to(grad.dtype)
        out.append((_f32(p), _f32(s1), None if s2 is None else _f32(s2)))
    nat.check()
    (pr, s1r, s2r), (po, s1o, s2o) = out
    # identical up to the contraction of an fma here and there (fp16 / bf16: bit-identical in practice)
    _close(po, pr, dtype, f"{name} {dtype}: p vs the reference library", ulps=2.01, atol=0, scale_ulps=2.0)
    _close(s1o, s1r, "fp32", f"{name}: state1 vs the reference library", ulps=4, atol=0, scale_ulps=4.0)
    if two:
        _close(s2o, s2r, "fp32", f"{name}: state2 vs the reference library", ulps=4, atol=0, scale_ulps=4.0)
    assert np.mean(po == pr) > 0.85  # (fp32 RMSprop: ~8 % of the parameters differ by an ulp, the rest of the table is > 97 %)
    print(f"{ours_sym}: p identical {np.mean(po == pr):.6f}, state1 identical {np.mean(s1o == s1r):.6f}")


@pytest.mark.parametrize("name", list(OPT_ID))
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("n", [65536, 1000])
def test_8bit_blockwise_update_equals_the_reference_cuda_library(name, dtype, n):
    if name == "ademamix" and n % 256:
        pytest.skip("the reference indexes the slow EMA's absmax at (n + i) / 256: defined for n % 256 == 0 only")
    ref = nat.ref_cuda()
    sym = f"c{name}_8bit_blockwise_grad_{dtype}"
    lr, b1, b2, b3, alpha, eps, wd = HYPER[name]
    code1, code2 = _codes()
    out = []
    for L in (ref, nat.lib):
        fn = getattr(L, sym)
        p, grad = _inputs(n, dtype, 31)
        c1, c2, a1, a2 = _blockwise_state(name, n, 9)
        for step in (1, 2, 3):
            torch.cuda.synchronize()
            fn(nat.ptr(p), nat.ptr(grad), nat.ptr(c1), nat.ptr(c2), b1, b2, b3, alpha, eps, step, lr, nat.ptr(code1),
               nat.ptr(code2) if c2 is not None else None, nat.ptr(a1), nat.ptr(a2), wd, 1.0, False, n)
            torch.cuda.synchronize()
            grad = (grad.float() * 0.7 - 0.02).to(grad.dtype)
        out.append((_f32(p), c1.cpu().numpy(), None if c2 is None else c2.cpu().numpy(), _f32(a1), None if a2 is None else _f32(a2)))
    nat.check()
    r, o = out
    same_p = np.mean(r[0] == o[0])
    same_c1 = np.mean(r[1] == o[1])
    print(f"{sym} n={n}: p identical {same_p:.6f}, state1 codes identical {same_c1:.6f}")
    np.testing.assert_allclose(o[3], r[3], rtol=1e-6, atol=1e-12, err_msg="absmax1")
    if r[4] is not None:
        np.testing.assert_allclose(o[4], r[4], rtol=1e-6, atol=1e-20, err_msg="absmax2")
        assert np.mean(r[2] == o[2]) > 0.999
    assert same_c1 > 0.999, f"state1 codes identical only at {same_c1}"
    _close(o[0], r[0], dtype, f"{name} {dtype}: p vs the reference library", ulps=2.01, atol=0, scale_ulps=2.0)


# ------------------------------------------------------------------------------------------ public classes
def _model(dtype=torch.float32, seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 32)).cuda().to(dtype)


def _train(model, opt, steps=40):
    g = torch.Generator(device="cpu").manual_seed(1)
    x = torch.randn(256, 64, generator=g).cuda().to(next(model.parameters()).dtype)
    y = torch.randn(256, 32, generator=g).cuda().to(x.dtype)
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        loss = torch.nn.functional.mse_loss(model(x), y)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    return losses


def _walk(make, steps=30, shape=(256, 96), seed=0):
    """The protocol of the reference's own optimizer test (reference tests/test_optim.py): one tensor, the SAME random
    gradient fed to every optimizer at every step, so that round-off does not feed back through a model."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    p = torch.nn.Parameter((torch.randn(shape, generator=g) * 0.1).cuda())
    opt = make([p])
    traj = []
    for _ in range(steps):
        p.grad = (torch.randn(shape, generator=g) * 0.01).cuda()
        opt.step()
        traj.append(p.detach().clone())
    return traj


def _pairs():
    import bitsandbytes_b200 as bnb

    O = bnb.optim
    return {
        "adam": (lambda ps: torch.optim.Adam(ps, lr=1e-3), lambda ps, bits: O.Adam(ps, lr=1e-3, optim_bits=bits, min_8bit_size=16)),
        "adamw": (lambda ps: torch.optim.AdamW(ps, lr=1e-3, weight_decay=0.05),
                  lambda ps, bits: O.AdamW(ps, lr=1e-3, weight_decay=0.05, optim_bits=bits, min_8bit_size=16)),
        "sgd": (lambda ps: torch.optim.SGD(ps, lr=1e-2, momentum=0.9),
                lambda ps, bits: O.SGD(ps, lr=1e-2, momentum=0.9, optim_bits=bits, min_8bit_size=16)),
        "rmsprop": (lambda ps: torch.optim.RMSprop(ps, lr=1e-3, alpha=0.99, eps=1e-8),
                    lambda ps, bits: O.RMSprop(ps, lr=1e-3, alpha=0.99, eps=1e-8, optim_bits=bits, min_8bit_size=16)),
        "adagrad": (lambda ps: torch.optim.Adagrad(ps, lr=1e-2, eps=1e-10),
                    lambda ps, bits: O.Adagrad(ps, lr=1e-2, optim_bits=bits, min_8bit_size=16)),
    }


@pytest.mark.parametrize("name", ["adam", "adamw", "sgd", "rmsprop", "adagrad"])
def test_public_optimizers_track_torch_optim(name):
    mk_torch, mk = _pairs()[name]
    want = _walk(mk_torch)
    got32 = _walk(lambda ps: mk(ps, 32))
    for step, (a, b) in enumerate(zip(want, got32)):
        torch.testing.assert_close(b, a, rtol=1e-5, atol=2e-6, msg=lambda m: f"{name} 32-bit, step {step}: {m}")
    got8 = _walk(lambda ps: mk(ps, 8))
    moved = float((want[-1] - want[0]).norm())
    off = float((got8[-1] - want[-1]).norm())
    assert off < 0.05 * moved, f"{name} 8-bit state: end point {off:.3e} away after a path of {moved:.3e}"


def test_lion_and_ademamix_8bit_follow_their_32bit_versions_and_train_a_model():
    import bitsandbytes_b200 as bnb

    makers = {"lion": lambda ps, bits: bnb.optim.Lion(ps, lr=1e-4, weight_decay=0.01, optim_bits=bits, min_8bit_size=16),
              "ademamix": lambda ps, bits: bnb.optim.AdEMAMix(ps, lr=1e-3, optim_bits=bits, min_8bit_size=16, t_alpha=20, t_beta3=20)}
    for name, mk in makers.items():
        a, b = _walk(lambda ps: mk(ps, 32)), _walk(lambda ps: mk(ps, 8))
        moved, off = float((a[-1] - a[0]).norm()), float((b[-1] - a[-1]).norm())
        assert off < 0.08 * moved, f"{name}: 8-bit end point {off:.3e} away after a path of {moved:.3e}"
        m = _model()
        losses = _train(m, mk(m.parameters(), 8), steps=60)
        assert losses[-1] < losses[0], f"{name} 8-bit does not reduce the loss"


def test_min_8bit_size_keeps_small_tensors_in_32_bits_and_state_dict_round_trips():
    import bitsandbytes_b200 as bnb

    m = _model()
    opt = bnb.optim.Adam8bit(m.parameters(), lr=1e-2)  # min_8bit_size 4096: the 128x64 weight is 8-bit, the biases are not
    _train(m, opt, steps=3)
    kinds = {tuple(p.shape): opt.state[p]["state1"].dtype for p in m.parameters()}
    assert kinds[(128, 64)] == torch.uint8 and kinds[(128,)] == torch.float32
    sd = opt.state_dict()
    wrapped = [v for v in sd["state"].values() if bnb.optim.Adam8bit._FSDP_WRAPPED_QUANT_STATE_KEY in v]
    assert wrapped, "the quantisation tensors travel under one wrapped key"
    m2 = _model()
    m2.load_state_dict(m.state_dict())
    opt2 = bnb.optim.Adam8bit(m2.parameters(), lr=1e-2)
    opt2.load_state_dict(sd)
    la, lb = _train(m, opt, steps=3), _train(m2, opt2, steps=3)
    assert la == lb, "a reloaded optimizer continues bit for bit"


def test_paged_optimizer_state_lives_in_managed_memory():
    import bitsandbytes_b200 as bnb

    torch.manual_seed(0)
    w = torch.nn.Parameter(torch.randn(512, 512, device="cuda"))  # >= 1e5 elements: paged
    opt = bnb.optim.PagedAdamW8bit([w], lr=1e-2)
    ref_w = torch.nn.Parameter(w.detach().clone())
    ref = bnb.optim.AdamW8bit([ref_w], lr=1e-2)
    for _ in range(3):
        for prm, o in ((w, opt), (ref_w, ref)):
            o.zero_grad()
            (prm.square().sum()).backward()
            o.step()
    assert getattr(opt.state[w]["state1"], "is_paged", False) and opt.state[w]["state1"].device.type == "cpu"
    assert torch.equal(w, ref_w), "paging changes where the state lives, not the update"
    assert torch.equal(opt.state[w]["state1"].cuda(), ref.state[ref_w]["state1"])
