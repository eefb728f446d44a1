"""Edge cases of the optimizer updates (csrc/optim.cu) that tests/test_gpu_optim.py does not reach.

Every case runs through the native entries (cbnb_b200_optimizer_update_32bit / _8bit_blockwise) and is compared with
two references:

* the numpy oracle (oracle/optim_ref.py), at the tolerances of tests/test_gpu_optim.py;
* the reference CUDA library built from the reference sources (tests/_native.ref_cuda(): same symbols, same buffers),
  at the agreement bars of test_gpu_optim.py's reference-library tests.  This comparison also pins the oracle's model
  of gnorm_scale, skip_zeros, non-finite gradients and the trust ratio, which tests/golden/reference_optim.npz does not
  cover.  The reference exports no bf16 momentum / RMSprop / Adagrad with 32-bit state; those cases have the oracle
  only.  Without a built reference library a test runs its oracle comparison and is then reported as skipped.

The cases:

* sizes past one wave of the persistent grid (8 CTAs per SM): 4096 x 4096 (+ 37) elements, so every CTA (32-bit state)
  and every warp (8-bit state) makes several passes; and one multi-tensor call over the LoRA set of a Llama-3-8B plus a
  4096 x 4096 weight, against the single-tensor calls;
* gnorm_scale != 1, also through the multi-tensor calls;
* skip_zeros = True, also through a public optimizer class;
* NaN and +-inf gradients;
* 8-bit blocks whose absmax is, or becomes, 0;
* the LAMB / LARS trust ratio (max_unorm > 0) at 16.8 M elements, and the public LAMB and LARS classes.
"""
import functools
import math

import numpy as np
import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.functional as F
from oracle import optim_ref as R
from tests import _native as nat
from tests.test_gpu_optim import HYPER, OPT_ID, _blockwise_state, _close, _codes, _f32, _inputs, _ref_name32
from tests.test_gpu_optim_multi import _assert_bits_equal, lora_shapes

pytestmark = pytest.mark.gpu

BIG = 4096 * 4096
SMALL = 12345  # 48 whole 256-element blocks and a ragged one of 57 elements; n % 4 == 1
TWO = ("adam", "ademamix")
COUPLED = ("momentum", "rmsprop", "adagrad")  # weight decay folds into the gradient
DTYPES = ["fp32", "fp16", "bf16"]


@functools.lru_cache(maxsize=None)
def _books():
    return _codes()


def _size(bits, name, n):
    """n, rounded down to a multiple of 256 for AdEMAMix's 8-bit state: the reference indexes its slow EMA's absmax at
    (n + i) / 256, which is defined for n % 256 == 0 only."""
    return n - n % 256 if bits == 8 and name == "ademamix" else n


def _bufs(bits, name, dtype, n, seed):
    """Parameters, gradients and a mid-training state: dict(p, g, s1, s2, a1, a2, n)."""
    p, g = _inputs(n, dtype, seed)
    if bits == 8:
        c1, c2, a1, a2 = _blockwise_state(name, n, seed + 1)
        return dict(p=p, g=g, s1=c1, s2=c2, a1=a1, a2=a2, n=n)
    gen = torch.Generator(device="cpu").manual_seed(seed + 1)
    s1 = (torch.rand((2, n) if name == "ademamix" else (n,), generator=gen) * 0.01).cuda()
    s2 = (torch.rand(n, generator=gen) * 0.001).cuda() if name in TWO else None
    return dict(p=p, g=g, s1=s1, s2=s2, a1=None, a2=None, n=n)


def _clone(t):
    return {k: v.clone() if isinstance(v, torch.Tensor) else v for k, v in t.items()}


def _gather32(t, sel):
    """The 4096-element chunks `sel` (ascending, a ragged last one last) of 32-bit-state buffers, as the buffers of one
    smaller tensor."""
    n = t["n"]
    chunks = torch.tensor(sel, device="cuda")
    elems = (chunks[:, None] * 4096 + torch.arange(4096, device="cuda")).reshape(-1)
    elems = elems[elems < n]
    s1 = t["s1"].reshape(-1, n)[:, elems]
    return dict(p=t["p"][elems], g=t["g"][elems], s1=s1 if s1.shape[0] == 2 else s1[0],
                s2=None if t["s2"] is None else t["s2"][elems], a1=None, a2=None, n=elems.numel())


def _gather8(t, sel):
    """The blocks `sel` (ascending, a ragged last block last) of 8-bit buffers, as the buffers of one smaller tensor.
    AdEMAMix's slow EMA keeps its layout: codes in the second row of state1, absmax after the first state's."""
    n, nb = t["n"], -(-t["n"] // 256)
    blocks = torch.tensor(sel, device="cuda")
    elems = (blocks[:, None] * 256 + torch.arange(256, device="cuda")).reshape(-1)
    elems = elems[elems < n]
    s1 = t["s1"].reshape(-1, n)[:, elems]
    a1 = t["a1"][blocks] if s1.shape[0] == 1 else torch.cat([t["a1"][blocks], t["a1"][nb + blocks]])
    pick = lambda v, i: None if v is None else v[i]  # noqa: E731
    return dict(p=t["p"][elems], g=t["g"][elems], s1=s1 if s1.shape[0] == 2 else s1[0], s2=pick(t["s2"], elems), a1=a1,
                a2=pick(t["a2"], blocks), n=elems.numel())


def _regrad(t, keep_zero=None):
    """The next step's gradient, a fixed function of this one; the elements under keep_zero stay 0."""
    g = t["g"].float() * 0.7 - 0.02
    if keep_zero is not None:
        g[keep_zero] = 0.0
    t["g"] = g.to(t["g"].dtype)


def _hyper(name, wd):
    lr, b1, b2, b3, alpha, eps, hwd = HYPER[name]
    return lr, b1, b2, b3, alpha, eps, hwd if wd is None else wd


def _ours(bits, name, dtype, t, step, log=None, gs=1.0, skip=False, wd=None, unorm=None, max_unorm=0.0, pn=0.0):
    """One step of t through this library's native entry.  log: a list that receives (step, arguments, inputs,
    outputs), for _vs_ref."""
    kw = dict(gs=gs, skip=skip, wd=wd, unorm=unorm, max_unorm=max_unorm, pn=pn)
    inputs = _clone(t) if log is not None else None
    lr, b1, b2, b3, alpha, eps, wd = _hyper(name, wd)
    P, n = nat.ptr, t["p"].numel()
    if bits == 32:
        rc = nat.lib.cbnb_b200_optimizer_update_32bit(OPT_ID[name], nat.DTYPE_ID[dtype], P(t["g"]), P(t["p"]), P(t["s1"]),
                                                      P(t["s2"]), P(unorm), max_unorm, pn, b1, b2, b3, alpha, eps, wd,
                                                      step, lr, gs, skip, n, nat.stream())
    else:
        code1, code2 = _books()
        rc = nat.lib.cbnb_b200_optimizer_update_8bit_blockwise(
            OPT_ID[name], nat.DTYPE_ID[dtype], P(t["p"]), P(t["g"]), P(t["s1"]), P(t["s2"]), b1, b2, b3, alpha, eps, step,
            lr, P(code1), P(code2) if t["s2"] is not None else None, P(t["a1"]), P(t["a2"]), wd, gs, skip, n, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    if log is not None:
        log.append((step, kw, inputs, _clone(t)))


def _multi(bits, name, ts, step, gs=1.0, skip=False, wd=None):
    """One step of every tensor of ts through the multi-tensor call."""
    lr, b1, b2, b3, alpha, eps, wd = _hyper(name, wd)
    two = name in TWO
    col = lambda k: [t[k] for t in ts]  # noqa: E731
    steps = [step] * len(ts)
    if bits == 8:
        code1, code2 = _books()
        F.optimizer_update_8bit_blockwise_multi(name, col("g"), col("p"), col("s1"), col("s2") if two else None, b1, b2, b3,
                                                alpha, eps, steps, lr, code1, code2 if two else None, col("a1"),
                                                col("a2") if two else None, wd, gnorm_scale=gs, skip_zeros=skip)
    else:
        F.optimizer_update_32bit_multi(name, col("g"), col("p"), col("s1"), b1, eps, steps, lr, col("s2") if two else None,
                                       b2, b3, alpha, wd, gnorm_scale=gs, skip_zeros=skip)
    torch.cuda.synchronize()
    nat.check()


def _has_ref(bits, name, dtype):
    return bits == 8 or _ref_name32(name, dtype) is not None


def _ref(bits, name, dtype, t, step, gs=1.0, skip=False, wd=None, unorm=None, max_unorm=0.0, pn=0.0):
    """The same step through the reference CUDA library (its symbols run on the legacy default stream)."""
    lr, b1, b2, b3, alpha, eps, wd = _hyper(name, wd)
    P, n = nat.ptr, t["p"].numel()
    ref = nat.ref_cuda()
    torch.cuda.synchronize()
    if bits == 32:
        getattr(ref, _ref_name32(name, dtype))(P(t["g"]), P(t["p"]), P(t["s1"]), P(t["s2"]), P(unorm), max_unorm, pn, b1,
                                               b2, b3, alpha, eps, wd, step, lr, gs, skip, n)
    else:
        code1, code2 = _books()
        getattr(ref, f"c{name}_8bit_blockwise_grad_{dtype}")(
            P(t["p"]), P(t["g"]), P(t["s1"]), P(t["s2"]), b1, b2, b3, alpha, eps, step, lr, P(code1),
            P(code2) if t["s2"] is not None else None, P(t["a1"]), P(t["a2"]), wd, gs, skip, n)
    torch.cuda.synchronize()


def _vs_ref(bits, name, dtype, log, what, elems=None, blocks=None, identical=0.85):
    """Every logged step again through the reference library, from the same inputs, against this library's outputs
    (_check_ref).  Step by step, so that a code one entry away (which the bars allow) does not move a later step.
    Returns the (ours, reference) buffers of each step."""
    pairs = []
    if not _has_ref(bits, name, dtype):
        return pairs
    for step, kw, inputs, out in log:
        r = _clone(inputs)
        if kw["unorm"] is not None:
            kw = dict(kw, unorm=torch.zeros(1, device="cuda"))
        _ref(bits, name, dtype, r, step, **kw)
        _check_ref(bits, dtype, out, r, f"{what} step {step}", elems, blocks, identical)
        pairs.append((out, r))
    return pairs


def _np(v):
    if v is None:
        return None
    return v.cpu().numpy() if v.dtype == torch.uint8 else _f32(v)


def _oracle(bits, name, dtype, t, step, gs=1.0, skip=False, wd=None, max_unorm=0.0):
    """The oracle's step from t's current values (t is not changed)."""
    lr, b1, b2, b3, alpha, eps, wd = _hyper(name, wd)
    args = (_np(t["g"]), _np(t["p"]), _np(t["s1"]), _np(t["s2"]))
    with np.errstate(all="ignore"):  # (non-finite gradients, 0 / 0 in a block whose absmax is 0)
        if bits == 32:
            return R.update_32bit(name, dtype, *args, step, lr, b1, b2, b3, alpha, eps, wd, gnorm_scale=gs,
                                  max_unorm=max_unorm, skip_zeros=skip)
        code1, code2 = _books()
        return R.update_8bit_blockwise(name, dtype, *args, code1.cpu().numpy(), code2.cpu().numpy(), _np(t["a1"]),
                                       _np(t["a2"]), step, lr, b1, b2, b3, alpha, eps, wd, gnorm_scale=gs, skip_zeros=skip)


def _check_oracle(bits, dtype, t, want, p_before, what):
    """The tolerances of test_gpu_optim.py's oracle tests.  Its 32-bit test starts from a zero state, so two allowances
    of its 8-bit test and of its reference-library bars carry over here to the 32-bit state:
    * the parameter may move by 2e-3 of its own update: the kernels' __powf (--use_fast_math) carries a relative error
      that 1 - __powf(beta2, step) magnifies up to ~1e-4, where the oracle's pow is exact; and it is rounded twice
      (after the update, after the decoupled weight decay), each time perhaps to the other side: 2 ulp;
    * a state may move by 2 ulp of the largest state: a mid-training state and the gradient term cancel, and an fma
      contracted differently moves the sum by an ulp of its larger term."""
    if bits == 32:
        upd = np.abs(want[0] - p_before)
        _close(_f32(t["p"]), want[0], dtype, f"{what}: p", ulps=2.01, atol=2e-3 * np.where(np.isfinite(upd), upd, 0))
        _close(_f32(t["s1"]), want[1], "fp32", f"{what}: state1", ulps=8, atol=1e-9, scale_ulps=2.0)
        if t["s2"] is not None:
            _close(_f32(t["s2"]), want[2], "fp32", f"{what}: state2", ulps=8, atol=1e-12, scale_ulps=2.0)
        return
    np.testing.assert_allclose(_f32(t["a1"]), want[3], rtol=2e-6, atol=1e-12, err_msg=f"{what}: absmax1")
    if t["a2"] is not None:
        np.testing.assert_allclose(_f32(t["a2"]), want[4], rtol=2e-6, atol=1e-20, err_msg=f"{what}: absmax2")
    upd = np.abs(want[0] - p_before)
    upd = upd[np.isfinite(upd)]
    _close(_f32(t["p"]), want[0], dtype, f"{what}: p", ulps=1.01, atol=2e-3 * float(upd.max()) if upd.size else 0.0)
    c1 = t["s1"].cpu().numpy()
    same1 = (c1 == want[1]).mean()
    assert same1 > 0.995, f"{what}: state1 codes agree only at {same1:.4f}"
    d1 = np.abs(c1.astype(np.int64) - want[1].astype(np.int64))
    assert d1.max() <= 1, f"{what}: a state1 code is {d1.max()} entries away from the oracle's"
    if t["s2"] is not None:
        same2 = (t["s2"].cpu().numpy() == want[2]).mean()
        assert same2 > 0.995, f"{what}: state2 codes agree only at {same2:.4f}"


def _same_nonfinite(got, want, what):
    """NaN where the reference has NaN, and the same infinities."""
    inf = np.isinf(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)), f"{what}: NaN at other elements"
    assert np.array_equal(np.isinf(got), inf) and np.array_equal(got[inf], want[inf]), f"{what}: other infinities"


def _check_ref(bits, dtype, o, r, what, elems=None, blocks=None, identical=0.85):
    """The bars of test_gpu_optim.py's reference-library tests, over the elements `elems` and the 8-bit blocks `blocks`
    (default: all); a non-finite value must be the same value.  `identical`: the share of bit-identical 32-bit-state
    parameters."""
    el = slice(None) if elems is None else elems
    bl = slice(None) if blocks is None else blocks
    po, pr = _f32(o["p"])[el], _f32(r["p"])[el]
    _same_nonfinite(po, pr, f"{what}: p")
    _close(po, pr, dtype, f"{what}: p vs the reference library", ulps=2.01, atol=0, scale_ulps=2.0)
    if bits == 32:
        for k in ("s1", "s2"):
            if o[k] is not None:
                so, sr = _f32(o[k]), _f32(r[k])
                _same_nonfinite(so, sr, f"{what}: {k}")
                _close(so, sr, "fp32", f"{what}: {k} vs the reference library", ulps=4, atol=0, scale_ulps=4.0)
        assert np.mean(po == pr) > identical, f"{what}: p identical only at {np.mean(po == pr):.4f}"
        return
    np.testing.assert_allclose(_f32(o["a1"])[bl], _f32(r["a1"])[bl], rtol=1e-6, atol=1e-12, err_msg=f"{what}: absmax1")
    if o["a2"] is not None:
        np.testing.assert_allclose(_f32(o["a2"])[bl], _f32(r["a2"])[bl], rtol=1e-6, atol=1e-20, err_msg=f"{what}: absmax2")
    for k in ("s1", "s2"):
        if o[k] is not None:
            same = np.mean(o[k].cpu().numpy()[..., el] == r[k].cpu().numpy()[..., el])
            assert same > 0.999, f"{what}: {k} codes identical to the reference's only at {same:.6f}"


def _bits(t):
    """Raw bits of a tensor (NaN payloads and the sign of 0 included)."""
    b = nat.to_bits(t)
    return b.view(np.uint32) if b.dtype == np.float32 else b


# ------------------------------------------------------------------------------------------ past one wave of the grid
WAVES = [(32, "adam"), (32, "lion"), (32, "ademamix"), (8, "adam"), (8, "momentum"), (8, "ademamix")]


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("bits,name", WAVES, ids=[f"{b}bit-{n}" for b, n in WAVES])
def test_updates_past_one_wave_of_the_persistent_grid(bits, name, dtype):
    """4096 x 4096 (+ 37) elements: each CTA (32-bit: 4096-element chunks) or warp (8-bit: 256-element blocks) takes
    several work items and finds their tensor again on each pass."""
    n = _size(bits, name, BIG + 37)
    per_item = 4096 if bits == 32 else 256
    items_per_wave = 8 * torch.cuda.get_device_properties(0).multi_processor_count * (1 if bits == 32 else 8)
    assert -(-n // per_item) > 3 * items_per_wave
    t = _bufs(bits, name, dtype, n, seed=41)
    log = []
    # the oracle costs a second or more per step at this size: it checks every 29th 4096-element chunk (about 36 per
    # pass of the grid) or every 61st 256-element block (about 140 per pass), and the ragged last one; the reference
    # library checks every element
    items = -(-n // per_item)
    sel = sorted(set(range(0, items, 29 if bits == 32 else 61)) | {items - 1})
    view = (lambda x: _gather32(x, sel)) if bits == 32 else (lambda x: _gather8(x, sel))
    for step in (2, 3):
        want, before = _oracle(bits, name, dtype, view(t), step), _f32(view(t)["p"])
        _ours(bits, name, dtype, t, step, log)
        _check_oracle(bits, dtype, view(t), want, before, f"{name} {dtype} {bits}-bit n={n} step {step}")
        _regrad(t)
    _vs_ref(bits, name, dtype, log, f"{name} {dtype} {bits}-bit n={n}")


@pytest.mark.parametrize("bits", [8, 32])
def test_a_multi_tensor_call_over_several_waves_equals_the_single_tensor_calls(bits):
    """The 448 LoRA tensors of a Llama-3-8B (r = 16) and one 4096 x 4096 weight: 58.7 M elements, each tensor at its own
    step, in one multi-tensor AdamW call, bit for bit the single-tensor calls."""
    gen = torch.Generator(device="cuda").manual_seed(7)
    ts = []
    for i, shape in enumerate(lora_shapes(16) + [(4096, 4096)]):
        n = math.prod(shape)
        nb = -(-n // 256)
        t = dict(n=n, step=1 + i % 7, p=(torch.randn(n, device="cuda", generator=gen) * 0.02).to(torch.bfloat16),
                 g=(torch.randn(n, device="cuda", generator=gen) * 1e-3).to(torch.bfloat16))
        if bits == 8:
            t.update(s1=torch.randint(0, 256, (n,), device="cuda", generator=gen, dtype=torch.uint8),
                     s2=torch.randint(0, 256, (n,), device="cuda", generator=gen, dtype=torch.uint8),
                     a1=torch.rand(nb, device="cuda", generator=gen) * 0.05 + 1e-3,
                     a2=torch.rand(nb, device="cuda", generator=gen) * 0.002 + 1e-5)
        else:
            t.update(s1=torch.rand(n, device="cuda", generator=gen) * 0.01,
                     s2=torch.rand(n, device="cuda", generator=gen) * 0.001, a1=None, a2=None)
        ts.append(t)
    per_item = 256 if bits == 8 else 4096
    items_per_wave = 8 * torch.cuda.get_device_properties(0).multi_processor_count * (8 if bits == 8 else 1)
    assert sum(-(-t["n"] // per_item) for t in ts) > 3 * items_per_wave
    single = [_clone(t) for t in ts]
    lr, b1, b2, b3, alpha, eps, wd = HYPER["adam"]
    col = lambda k: [t[k] for t in ts]  # noqa: E731
    if bits == 8:
        code1, code2 = _books()
        F.optimizer_update_8bit_blockwise_multi("adam", col("g"), col("p"), col("s1"), col("s2"), b1, b2, b3, alpha, eps,
                                                col("step"), lr, code1, code2, col("a1"), col("a2"), wd)
    else:
        F.optimizer_update_32bit_multi("adam", col("g"), col("p"), col("s1"), b1, eps, col("step"), lr, col("s2"), b2, b3,
                                       alpha, wd)
    torch.cuda.synchronize()
    nat.check()
    for t in single:
        _ours(bits, "adam", "bf16", t, t["step"])
    for i, (a, b) in enumerate(zip(ts, single)):
        _assert_bits_equal(a, b, f"adam {bits}-bit, tensor {i} of {len(ts)}")


# ------------------------------------------------------------------------------------------ gnorm_scale
@pytest.mark.parametrize("gs", [0.25, 3.0])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(OPT_ID))
@pytest.mark.parametrize("bits", [32, 8])
def test_gnorm_scale(bits, name, dtype, gs):
    """The gradient is scaled by gnorm_scale: rounded to its dtype in the 32-bit kernels, in fp32 in the 8-bit ones,
    where the one-state RMSprop / Adagrad parameter update divides the UNSCALED gradient (as the reference).  The
    multi-tensor call (a list of two, so not the single-tensor instance) gives the single-tensor bits.

    8-bit RMSprop / Adagrad divide that unscaled gradient by the root of a state built from gnorm_scale * g +
    weight_decay * p.  Where the two terms cancel to under 1/20 of the first, an ulp of either moves the step by 20 ulp
    or more, so there the comparison with the reference library is left to the oracle's bound, which scales with the
    update."""
    n = _size(bits, name, SMALL)
    t = _bufs(bits, name, dtype, n, seed=51)
    extra = _bufs(bits, name, dtype, _size(bits, name, 1000), seed=52)
    t_multi, extra_single, log = _clone(t), _clone(extra), []
    what = f"{name} {dtype} {bits}-bit gnorm_scale {gs}"
    for step in (2, 3):
        want, before = _oracle(bits, name, dtype, t, step, gs=gs), _f32(t["p"])
        _ours(bits, name, dtype, t, step, log, gs=gs)
        _check_oracle(bits, dtype, t, want, before, f"{what} step {step}")
        _ours(bits, name, dtype, extra_single, step, gs=gs)
        _multi(bits, name, [t_multi, extra], step, gs=gs)
        _assert_bits_equal(t_multi, t, f"{what} step {step}: multi-tensor call")
        _assert_bits_equal(extra, extra_single, f"{what} step {step}: multi-tensor call, second tensor")
        for x in (t, t_multi, extra, extra_single):
            _regrad(x)
    elems = None
    if bits == 8 and name in ("rmsprop", "adagrad"):
        wd = HYPER[name][6]
        elems = np.ones(n, bool)
        for _, _, inputs, _ in log:
            term = _f32(inputs["g"]) * np.float32(gs)
            elems &= np.abs(term + _f32(inputs["p"]) * np.float32(wd)) >= 0.05 * np.abs(term)
        assert elems.mean() > 0.95
    _vs_ref(bits, name, dtype, log, what, elems=elems)


# ------------------------------------------------------------------------------------------ coupled weight decay
def _cancelling(dtype, wd, count):
    """`count` parameters p of `dtype` whose product p * wd, rounded to fp32, is itself a value of `dtype` (and not
    exact): with g = -fl32(p * wd), two roundings leave g + p * wd = 0, one leaves a residue."""
    if dtype == "fp32":
        p = np.random.default_rng(3).standard_normal(count).astype(np.float32)
    else:
        bits = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
        vals = (bits.view(np.float16).astype(np.float32) if dtype == "fp16"
                else (bits.astype(np.uint32) << 16).view(np.float32))
        vals = vals[np.isfinite(vals) & (np.abs(vals) > 0.05) & (np.abs(vals) < 2)]
        prod = vals * np.float32(wd)
        p = vals[(R._round_to(prod, dtype) == prod) & (prod.astype(np.float64) != vals.astype(np.float64) * np.float32(wd))]
        p = np.resize(p, count)
    prod = p * np.float32(wd)
    assert (prod.astype(np.float64) != p.astype(np.float64) * np.float32(wd)).all()
    return p, -prod


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("name", COUPLED)
def test_coupled_weight_decay_that_cancels_the_gradient(name, dtype):
    """Coupled weight decay folds into the gradient as one fused multiply-add, g + p * wd rounded once, in both CUDA
    libraries.  Where the gradient is -fl32(p * wd), the fold leaves a residue of the size of an fp32 rounding error,
    which Adagrad and RMSprop divide by its own magnitude: from a zero state, a step of about lr (Adagrad) where two
    roundings would leave 0 and no step.  Every other element of the tensor has such a gradient.  (In fp16 the residue
    is below the smallest subnormal, so both give 0.)

    The reference library's fp32 one-state kernel is not consistent here: its SASS folds element 0 of each thread's
    four as fma(p, wd, g * gnorm_scale) and elements 1 to 3 as fma(g, gnorm_scale, fl(p * wd)), which loses the
    residue.  The comparison with it covers the elements i % 4 == 0 and the elements without cancellation."""
    wd = HYPER[name][6]
    n = SMALL
    t = _bufs(32, name, dtype, n, seed=121)
    t["s1"].zero_()
    half = np.arange(0, n, 2)
    pv, gv = _cancelling(dtype, wd, half.size)
    t["p"][torch.from_numpy(half).cuda()] = torch.from_numpy(pv).cuda().to(t["p"].dtype)
    t["g"][torch.from_numpy(half).cuda()] = torch.from_numpy(gv).cuda().to(t["g"].dtype)
    log = []
    what = f"{name} {dtype} weight decay cancelling the gradient"
    want, before = _oracle(32, name, dtype, t, 1), _f32(t["p"])
    _ours(32, name, dtype, t, 1, log)
    _check_oracle(32, dtype, t, want, before, what)
    assert (_f32(t["s1"])[half] != 0).all(), f"{what}: a state holds no residue"
    _vs_ref(32, name, dtype, log, what, elems=np.arange(n) % 4 != 2)


# ------------------------------------------------------------------------------------------ skip_zeros
def _zero_mask(n):
    """Where the gradient is zeroed: every 7th element of the first half of the 256-element blocks, and all of block 2.
    The second half of the blocks has no zero."""
    nb = -(-n // 256)
    i = np.arange(n)
    m = (i % 7 == 3) & (i // 256 < nb // 2)
    m[512:768] = True
    return torch.from_numpy(m).cuda()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(OPT_ID))
def test_32bit_skip_zeros(name, dtype):
    """An element whose gradient is 0 keeps its parameter and state bits.  The test is made on the gradient after
    coupled weight decay (reference csrc/kernels.cu:859-871), which is 0 only where p * weight_decay cancels it, so
    momentum / RMSprop / Adagrad run without weight decay here.  AdEMAMix ignores the flag, as the reference does
    (csrc/kernels.cu:683-699): its steps are bit-equal to skip_zeros=False.  With the flag set, the two libraries round
    fp32 Lion's decay-then-sign step differently: a quarter of the parameters are an ulp apart (within the 2-ulp bar),
    so the share of identical parameters is held at 0.7 there."""
    wd = 0.0 if name in COUPLED else None
    zero = _zero_mask(SMALL)
    t = _bufs(32, name, dtype, SMALL, seed=61)
    t["g"][zero] = 0
    plain, log = _clone(t), []
    what = f"{name} {dtype} 32-bit skip_zeros"
    for step in (2, 3):
        want, before = _oracle(32, name, dtype, t, step, skip=True, wd=wd), _f32(t["p"])
        kept = {k: _bits(t[k])[..., zero.cpu().numpy()] for k in ("p", "s1", "s2") if t[k] is not None}
        _ours(32, name, dtype, t, step, log, skip=True, wd=wd)
        _check_oracle(32, dtype, t, want, before, f"{what} step {step}")
        if name == "ademamix":
            _ours(32, name, dtype, plain, step, wd=wd)
            _assert_bits_equal(t, plain, f"{what} step {step}: AdEMAMix ignores skip_zeros")
            _regrad(plain, zero)
        else:
            for k, b in kept.items():
                assert np.array_equal(_bits(t[k])[..., zero.cpu().numpy()], b), f"{what} step {step}: a skipped {k} changed"
        _regrad(t, zero)
    _vs_ref(32, name, dtype, log, what, identical=0.7 if name == "lion" else 0.85)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(OPT_ID))
def test_8bit_skip_zeros(name, dtype):
    """One-state optimizers: an element whose gradient is 0 keeps its parameter bits and its state value, which is
    requantised under the block's new absmax (optim.cu, as the oracle).  The zero test reads the raw gradient, before
    weight decay.  The reference's one-state kernel leaves a skipped element's state register unassigned
    (csrc/kernels.cu:1225-1261), so there a block with a skipped element has no defined absmax or codes: the comparison
    with it covers the blocks without zeros, and the oracle covers the rest (the elements past n of a ragged last
    block are zero gradients too).  Two-state optimizers ignore the flag, as
    the reference's kernel does: bit-equal to skip_zeros=False, and compared with the reference everywhere."""
    n = _size(8, name, SMALL)
    zero = _zero_mask(n)
    zn = zero.cpu().numpy()
    two = name in TWO
    t = _bufs(8, name, dtype, n, seed=71)
    t["g"][zero] = 0
    plain, log = _clone(t), []
    what = f"{name} {dtype} 8-bit skip_zeros"
    for step in (2, 3):
        want, before = _oracle(8, name, dtype, t, step, skip=True), _f32(t["p"])
        kept = _bits(t["p"])[zn]
        _ours(8, name, dtype, t, step, log, skip=True)
        _check_oracle(8, dtype, t, want, before, f"{what} step {step}")
        if two:
            _ours(8, name, dtype, plain, step)
            _assert_bits_equal(t, plain, f"{what} step {step}: the two-state kernel ignores skip_zeros")
            _regrad(plain, zero)
        else:
            assert np.array_equal(_bits(t["p"])[zn], kept), f"{what} step {step}: a skipped parameter changed"
        _regrad(t, zero)
    if two:
        _vs_ref(8, name, dtype, log, what)
        return
    dirty = np.zeros(-(-n // 256), bool)
    dirty[np.nonzero(zn)[0] // 256] = True
    dirty[-1] |= n % 256 != 0
    clean = ~dirty[np.arange(n) // 256]
    for o, r in _vs_ref(8, name, dtype, log, f"{what}, blocks without zeros", elems=clean, blocks=~dirty):
        same = np.mean(o["s1"].cpu().numpy()[~clean] == r["s1"].cpu().numpy()[~clean])
        print(f"{what}: state codes in the blocks with zeros identical to the reference's at {same:.4f}")


def test_skip_zeros_through_the_public_sgd_class():
    """SGD with momentum, 8-bit state and skip_zeros (given, as in the reference, through `args`): three steps from a
    fresh state equal the native single-tensor calls bit for bit, and skipped parameters do not move."""
    from bitsandbytes_b200.optim.optimizer import MockArgs

    lr, b1, b2, b3, alpha, eps, wd = HYPER["momentum"]
    shape = (64, 257)
    n = math.prod(shape)
    nb = -(-n // 256)
    zero = _zero_mask(n)
    gen = torch.Generator(device="cpu").manual_seed(5)
    w = torch.nn.Parameter((torch.randn(shape, generator=gen) * 0.1).cuda())
    args = MockArgs(dict(optim_bits=8, min_8bit_size=4096, max_unorm=0.0, skip_zeros=True))
    opt = bnb.optim.SGD([w], lr=lr, momentum=b1, weight_decay=wd, args=args)
    t = dict(p=w.detach().clone().reshape(-1), g=None, s1=torch.zeros(n, dtype=torch.uint8, device="cuda"), s2=None,
             a1=torch.zeros(nb, device="cuda"), a2=None, n=n)
    kept = _bits(w)[zero.cpu().numpy().reshape(shape)]
    for step in (1, 2, 3):
        g = (torch.randn(n, generator=gen) * 0.01).cuda()
        g[zero] = 0
        w.grad = g.reshape(shape).clone()
        t["g"] = g
        opt.step()
        _ours(8, "momentum", "fp32", t, step, skip=True)
        st = opt.state[w]
        assert st["state1"].dtype == torch.uint8 and st["step"] == step
        got = dict(p=w.detach().reshape(-1), s1=st["state1"].reshape(-1), s2=None, a1=st["absmax1"], a2=None, n=n)
        _assert_bits_equal(got, t, f"SGD 8-bit skip_zeros step {step} vs the native call")
        assert np.array_equal(_bits(w)[zero.cpu().numpy().reshape(shape)], kept), "a skipped parameter moved"


# ------------------------------------------------------------------------------------------ non-finite gradients
def _nonfinite(n):
    """(index, value): a NaN in the middle of a lane's 8-element group (and of a 4-element group of the 32-bit kernel),
    infinities at the two ends of a block, and three in the last block, which is ragged unless n % 256 == 0."""
    last = (n - 1) // 256 * 256
    return [(3 * 256 + 45, math.nan), (7 * 256 + 98, math.inf), (7 * 256 + 255, -math.inf), (last + 21, math.nan),
            (last + 1, math.inf), (n - 1, -math.inf)]


def _decode(codes, absmax, code, blk):
    return code.cpu().numpy()[codes.cpu().numpy()] * _f32(absmax)[blk]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(OPT_ID))
@pytest.mark.parametrize("bits", [32, 8])
def test_non_finite_gradients(bits, name, dtype):
    """NaN, +inf and -inf gradient elements.

    8-bit Adam / AdEMAMix guard them (reference csrc/kernels.cu:1017-1041, 1092): the element's parameter keeps its
    bits, its states are set to 0 (and decode to 0), and the rest of the block follows the oracle, as does the next,
    finite step.

    The 32-bit kernels and the 8-bit one-state kernels have no guard; they must do what the reference library does.
    After one step both libraries hold, at the non-finite gradients:
    * 32-bit Adam, AdEMAMix, momentum, RMSprop, Adagrad: a NaN or infinite state and a non-finite parameter;
    * 32-bit Lion: a non-finite state, and a parameter moved by lr * sign (0 for NaN), so finite;
    * 8-bit momentum, RMSprop, Adagrad, Lion: an infinite state makes its block's absmax infinite, so every state of
      that block decodes to 0 * inf = NaN in the next step; a NaN state is left out of the absmax.
    The comparison is exact at those elements (NaN for NaN, the same infinity, and the same codes) and at the bars of
    the reference-library tests elsewhere."""
    n = _size(bits, name, SMALL)
    pos = _nonfinite(n)
    idx = np.array([i for i, _ in pos])
    t = _bufs(bits, name, dtype, n, seed=81)
    for i, v in pos:
        t["g"][i] = v
    what = f"{name} {dtype} {bits}-bit non-finite gradients"
    guarded = bits == 8 and name in TWO
    p_bits = _bits(t["p"])[idx]
    log = []
    want, before = _oracle(bits, name, dtype, t, 2), _f32(t["p"])
    _ours(bits, name, dtype, t, 2, log)
    if guarded:
        _check_oracle(bits, dtype, t, want, before, f"{what} step 2")
        assert np.array_equal(_bits(t["p"])[idx], p_bits), f"{what}: a parameter with a non-finite gradient changed"
        code1, code2 = _books()
        blk = idx // 256
        c1 = t["s1"].reshape(-1, n)
        assert (_decode(c1[0][idx], t["a1"], code1, blk) == 0).all(), f"{what}: state1 does not decode to 0"
        assert (_decode(t["s2"][idx], t["a2"], code2, blk) == 0).all(), f"{what}: state2 does not decode to 0"
        if name == "ademamix":
            assert (_decode(c1[1][idx], t["a1"], code1, n // 256 + blk) == 0).all(), f"{what}: the slow EMA is not 0"
        _regrad(t)
        t["g"][idx] = 0.01
        want, before = _oracle(bits, name, dtype, t, 3), _f32(t["p"])
        _ours(bits, name, dtype, t, 3, log)
        _check_oracle(bits, dtype, t, want, before, f"{what} step 3 (finite gradients)")
    pairs = _vs_ref(bits, name, dtype, log, what)
    if pairs:
        o, r = pairs[0]
        for k in ("p", "s1", "s2"):
            if r[k] is not None:
                a, b = (_bits(x[k]).reshape(-1, n)[:, idx] for x in (o, r))
                assert np.array_equal(a, b), f"{what}: {k} at the non-finite gradients {a} != the reference's {b}"


# ------------------------------------------------------------------------------------------ absmax 0
@pytest.mark.parametrize("start", ["fresh", "mid-training"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(OPT_ID))
def test_8bit_blocks_whose_absmax_is_zero(name, dtype, start):
    """A block whose new absmax is 0 quantises 0 / 0 = NaN: its codes must be the reference library's (a stale or
    garbage code would carry into the next step), and the next step must stay finite and follow the oracle.

    `fresh`: the first step from the state init_state creates (codes 0, absmax 0), so every block decodes under an
    absmax of 0.  `mid-training`: one block of a mid-training state has absmax 0.  In both, block 5's gradients are 0,
    so its absmax stays 0 (momentum / RMSprop / Adagrad without weight decay, which would fold p * weight_decay into
    the gradient)."""
    n = _size(8, name, SMALL)
    nb, k = -(-n // 256), 5
    two = name in TWO
    wd = 0.0 if name in COUPLED else None
    t = _bufs(8, name, dtype, n, seed=91)
    if start == "fresh":
        for key in ("s1", "s2", "a1", "a2"):
            if t[key] is not None:
                t[key].zero_()
    else:
        t["a1"][k] = 0
        if two:
            t["a2"][k] = 0
        if name == "ademamix":
            t["a1"][nb + k] = 0
    t["g"][k * 256:(k + 1) * 256] = 0
    log = []
    step = 1 if start == "fresh" else 2
    what = f"{name} {dtype} {start}"
    zero_absmax = [("a1", k)] + ([("a2", k)] if two else []) + ([("a1", nb + k)] if name == "ademamix" else [])
    want, before = _oracle(8, name, dtype, t, step, wd=wd), _f32(t["p"])
    _ours(8, name, dtype, t, step, log, wd=wd)
    for key, b in zero_absmax:
        assert float(t[key][b]) == 0.0, f"{what}: {key}[{b}] is {float(t[key][b])}, not 0"
    _check_oracle(8, dtype, t, want, before, f"{what} step {step}")
    _regrad(t)
    want, before = _oracle(8, name, dtype, t, step + 1, wd=wd), _f32(t["p"])
    _ours(8, name, dtype, t, step + 1, log, wd=wd)
    for key in ("p", "a1", "a2"):
        if t[key] is not None:
            assert torch.isfinite(t[key]).all(), f"{what} step {step + 1}: {key} is not finite"
    _check_oracle(8, dtype, t, want, before, f"{what} step {step + 1}")
    o, r = _vs_ref(8, name, dtype, log, what)[0]
    blk = slice(k * 256, (k + 1) * 256)
    for key in ("s1", "s2"):
        if r[key] is not None:
            a, b = (x[key].reshape(-1, n)[:, blk].cpu().numpy() for x in (o, r))
            assert np.array_equal(a, b), f"{what}: {key} codes of the absmax-0 block differ from the reference's"
    for key, b in zero_absmax:
        assert float(r[key][b]) == 0.0


# ------------------------------------------------------------------------------------------ trust ratio
def _param_norm(p):
    """The oracle's parameter norm: float64, rounded to fp32."""
    return float(np.float32(np.linalg.norm(_f32(p).astype(np.float64))))


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("name", ["adam", "momentum", "rmsprop", "adagrad"])
def test_trust_ratio_at_16m_elements(name, dtype):
    """LAMB (adam) / LARS (momentum) / RMSprop / Adagrad with max_unorm > 0 at 4096 x 4096 + 37 elements, three steps.

    unorm is within 1e-4 of the oracle's float64 sum.  Every term of the sum is a square, so the relative error of an
    fp32 sum of them is at most (additions on the longest path) x 2^-24.  Here the pre-pass has 8 x 132 = 1056 CTAs of
    512 threads: a thread adds at most 32 terms, the warp and CTA reductions take 5 + 5 levels, and the CTAs' atomicAdd
    chain on unorm is at most 1056 long, in whatever order they land: at most 1098 x 2^-24 = 6.5e-5 in all.  The step
    is scaled by sqrt(max_unorm * param_norm / unorm), which is then within 3.3e-5 of the oracle's, well inside the
    2e-3 of its own update that _check_oracle allows a parameter."""
    n, max_unorm = BIG + 37, 0.01
    p, g = _inputs(n, dtype, 101)
    t = dict(p=p, g=g, s1=torch.zeros(n, device="cuda"), s2=torch.zeros(n, device="cuda") if name == "adam" else None,
             a1=None, a2=None, n=n)
    unorm, log = torch.zeros(1, device="cuda"), []
    what = f"{name} {dtype} max_unorm"
    for step in (1, 2, 3):
        pn = _param_norm(t["p"])
        want, before = _oracle(32, name, dtype, t, step, max_unorm=max_unorm), _f32(t["p"])
        assert math.sqrt(want[3]) > max_unorm * pn, f"{what}: the update norm is not clipped"
        _ours(32, name, dtype, t, step, log, unorm=unorm, max_unorm=max_unorm, pn=pn)
        got = float(unorm)
        assert abs(got - float(want[3])) <= 1e-4 * float(want[3]), f"{what} step {step}: unorm {got} vs {float(want[3])}"
        _check_oracle(32, dtype, t, want, before, f"{what} step {step}")
        _regrad(t)
    _vs_ref(32, name, dtype, log, what)


@pytest.mark.parametrize("cls", ["LAMB", "LARS"])
def test_public_lamb_and_lars_follow_the_oracle_step_by_step(cls):
    """Ten steps of the public class on a 1024 x 1024 parameter, each against optim_ref.update_32bit("lamb" | "lars")
    from the class's own state before the step: the parameter norm the class computes, its state and step counter, and
    the trust ratio it passes to the kernel, with the bounds of test_trust_ratio_at_16m_elements."""
    gen = torch.Generator(device="cpu").manual_seed(111)
    w = torch.nn.Parameter((torch.randn(1024, 1024, generator=gen) * 0.1).cuda())
    if cls == "LAMB":
        lr, b1, b2, eps, wd, mu = 1e-3, 0.9, 0.999, 1e-8, 0.01, 1.0
        opt = bnb.optim.LAMB([w], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, max_unorm=mu)
    else:
        lr, b1, b2, eps, wd, mu = 1e-2, 0.9, 0.0, 0.0, 1e-4, 0.02
        opt = bnb.optim.LARS([w], lr=lr, momentum=b1, weight_decay=wd, max_unorm=mu)
    n = w.numel()
    for step in range(1, 11):
        w.grad = (torch.randn(1024, 1024, generator=gen) * 0.01).cuda()
        st = opt.state[w]
        s1 = _f32(st["state1"]).reshape(-1) if "state1" in st else np.zeros(n, np.float32)
        s2 = (_f32(st["state2"]).reshape(-1) if "state2" in st else np.zeros(n, np.float32)) if cls == "LAMB" else None
        before = _f32(w).reshape(-1)
        want = R.update_32bit(cls.lower(), "fp32", _f32(w.grad).reshape(-1), before, s1, s2, step, lr, b1, b2, 0.0, 0.0, eps,
                              wd, max_unorm=mu)
        pn = float(np.linalg.norm(before.astype(np.float64)))
        assert math.sqrt(want[3]) > mu * pn, f"{cls} step {step}: the update norm is not clipped"
        opt.step()
        torch.cuda.synchronize()
        st = opt.state[w]
        what = f"{cls} step {step}"
        assert st["step"] == step
        got = float(st["unorm_vec"])
        assert abs(got - float(want[3])) <= 1e-4 * float(want[3]), f"{what}: unorm {got} vs {float(want[3])}"
        got = dict(p=w.detach().reshape(-1), s1=st["state1"].reshape(-1), s2=st["state2"].reshape(-1) if cls == "LAMB" else None)
        _check_oracle(32, "fp32", got, want, before, what)
