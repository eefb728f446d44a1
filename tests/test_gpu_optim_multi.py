"""GPU tests of the multi-tensor optimizer steps (csrc/optim.cu tensor lists, ``F.optimizer_update_*_multi`` and the
grouped ``Optimizer8bit.step``):

* one multi call over a ragged list equals, bit for bit, one single-tensor call per tensor on copies of the inputs,
  and the reference CUDA library's per-tensor symbols to the strictness of tests/test_gpu_optim.py (8-bit state:
  codes, absmax and 16-bit parameters identical; 32-bit state: within 2 ulp);
* a list longer than one launch's descriptor capacity;
* every optimizer class, 8- and 32-bit, against the per-parameter loop (update_step per parameter) on a model with
  many small parameters, bit for bit after every step;
* the number of optimizer kernels one step of AdamW8bit launches over the 448 LoRA tensors of a Llama-3-8B.
"""
import math

import numpy as np
import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.functional as F
from bitsandbytes_b200.backends.cuda import optimizer_multi_capacity
from tests import _native as nat
from tests.test_gpu_optim import HYPER, OPT_ID, _close, _codes, _ref_name32

pytestmark = pytest.mark.gpu

# ragged sizes (1 .. 65539); AdEMAMix's 8-bit slow EMA indexes its absmax at (n + i) / 256, which is defined (and free
# of a write race between the two halves) for n % 256 == 0 only, so its 8-bit list keeps to those sizes
SIZES = [1, 7, 255, 256, 257, 1000, 4096, 65539, 3, 512, 2048, 300, 4097, 17, 8192, 129, 1023, 5000, 64, 250, 768, 31]
SIZES_256 = [256, 512, 768, 1024, 4096, 65536, 256, 1280, 2048, 256, 512, 8192, 768, 256, 3072, 1024, 256, 512, 2304,
             256, 4352, 512]
MISALIGNED_P = 3  # p and g of this tensor start one element into their buffers
MISALIGNED_S = 5  # and state1 of this one


def _view(n_total, dtype, offset, fill):
    """A contiguous [n_total] view starting `offset` elements into a fresh buffer."""
    buf = fill(n_total + offset, dtype)
    return buf[offset:offset + n_total]


def _list(name, dtype, bits, seed):
    """Per tensor: dict(p, g, s1, s2, a1, a2, n, step) with random mid-training state."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    tdt = nat.DTYPE[dtype]
    two = name in ("adam", "ademamix")
    rows = 2 if name == "ademamix" else 1
    sizes = SIZES_256 if (name == "ademamix" and bits == 8) else SIZES
    out = []
    for i, n in enumerate(sizes):
        offp = 1 if i == MISALIGNED_P else 0
        offs = 1 if i == MISALIGNED_S else 0
        p = _view(n, tdt, offp, lambda m, d: (torch.randn(m, generator=gen) * 0.5).to(d).cuda())
        g = _view(n, tdt, offp, lambda m, d: (torch.randn(m, generator=gen) * 0.1).to(d).cuda())
        if bits == 8:
            nb = -(-n // 256)
            lo = 128 if name in ("rmsprop", "adagrad") else 0  # a second-moment state is never negative
            s1 = _view(rows * n, torch.uint8, offs,
                       lambda m, d: torch.randint(lo, 256, (m,), generator=gen, dtype=d).cuda())
            s2 = torch.randint(0, 256, (n,), generator=gen, dtype=torch.uint8).cuda() if two else None
            a1 = (torch.rand(rows * nb, generator=gen) * 0.05 + 1e-3).cuda()
            a2 = (torch.rand(nb, generator=gen) * 0.002 + 1e-5).cuda() if two else None
        else:
            s1 = _view(rows * n, torch.float32, offs, lambda m, d: (torch.rand(m, generator=gen) * 0.01).cuda())
            s2 = (torch.rand(n, generator=gen) * 0.001).cuda() if two else None
            a1 = a2 = None
        out.append(dict(p=p, g=g, s1=s1, s2=s2, a1=a1, a2=a2, n=n, step=1 + (i * 5) % 11))
    return out


def _copy(t):
    """A copy at the same storage offset: the same alignment, so the same vector or scalar path (for 16-bit parameters
    they round fp32 state differently: an fma contracted differently)."""
    off = t.storage_offset()
    out = torch.empty(t.numel() + off, dtype=t.dtype, device=t.device)[off:]
    return out.copy_(t)


def _clone(ts, aligned=False):
    cp = (lambda v: v.clone()) if aligned else _copy
    return [{k: (cp(v) if isinstance(v, torch.Tensor) else v) for k, v in t.items()} for t in ts]


def _multi(name, dtype, bits, ts, code1, code2):
    lr, b1, b2, b3, alpha, eps, wd = HYPER[name]
    two = ts[0]["s2"] is not None
    col = lambda k: [t[k] for t in ts]  # noqa: E731
    if bits == 8:
        F.optimizer_update_8bit_blockwise_multi(name, col("g"), col("p"), col("s1"), col("s2") if two else None, b1, b2, b3,
                                                alpha, eps, col("step"), lr, code1, code2 if two else None, col("a1"),
                                                col("a2") if two else None, wd)
    else:
        F.optimizer_update_32bit_multi(name, col("g"), col("p"), col("s1"), b1, eps, col("step"), lr,
                                       col("s2") if two else None, b2, b3, alpha, wd)


def _single(name, dtype, bits, ts, code1, code2):
    """One single-tensor native call per tensor (the stream-taking entries)."""
    lr, b1, b2, b3, alpha, eps, wd = HYPER[name]
    for t in ts:
        two = t["s2"] is not None
        if bits == 8:
            rc = nat.lib.cbnb_b200_optimizer_update_8bit_blockwise(
                OPT_ID[name], nat.DTYPE_ID[dtype], nat.ptr(t["p"]), nat.ptr(t["g"]), nat.ptr(t["s1"]), nat.ptr(t["s2"]), b1,
                b2, b3, alpha, eps, t["step"], lr, nat.ptr(code1), nat.ptr(code2) if two else None, nat.ptr(t["a1"]),
                nat.ptr(t["a2"]), wd, 1.0, False, t["n"], nat.stream())
        else:
            rc = nat.lib.cbnb_b200_optimizer_update_32bit(
                OPT_ID[name], nat.DTYPE_ID[dtype], nat.ptr(t["g"]), nat.ptr(t["p"]), nat.ptr(t["s1"]), nat.ptr(t["s2"]), None,
                0.0, 0.0, b1, b2, b3, alpha, eps, wd, t["step"], lr, 1.0, False, t["n"], nat.stream())
        assert rc == 0


def _reference(name, dtype, bits, ts, code1, code2):
    """The reference CUDA library's per-tensor symbols (legacy default stream).  Returns False where it has none."""
    ref = nat.ref_cuda()
    lr, b1, b2, b3, alpha, eps, wd = HYPER[name]
    if bits == 8:
        fn = getattr(ref, f"c{name}_8bit_blockwise_grad_{dtype}")
    else:
        sym = _ref_name32(name, dtype)
        if sym is None:  # (no bf16 momentum / RMSprop / Adagrad in the reference ABI)
            return False
        fn = getattr(ref, sym)
    torch.cuda.synchronize()
    for t in ts:
        two = t["s2"] is not None
        if bits == 8:
            fn(nat.ptr(t["p"]), nat.ptr(t["g"]), nat.ptr(t["s1"]), nat.ptr(t["s2"]), b1, b2, b3, alpha, eps, t["step"], lr,
               nat.ptr(code1), nat.ptr(code2) if two else None, nat.ptr(t["a1"]), nat.ptr(t["a2"]), wd, 1.0, False, t["n"])
        else:
            fn(nat.ptr(t["g"]), nat.ptr(t["p"]), nat.ptr(t["s1"]), nat.ptr(t["s2"]), None, 0.0, 0.0, b1, b2, b3, alpha, eps,
               wd, t["step"], lr, 1.0, False, t["n"])
    torch.cuda.synchronize()
    return True


def _assert_bits_equal(a, b, what):
    for k in ("p", "s1", "s2", "a1", "a2"):
        if a[k] is None:
            continue
        x, y = nat.to_bits(a[k]), nat.to_bits(b[k])
        if x.dtype == np.float32:
            x, y = x.view(np.uint32), y.view(np.uint32)
        bad = int((x != y).sum())
        assert bad == 0, f"{what}: {k} differs in {bad} of {x.size} elements (n = {a['n']})"


@pytest.mark.parametrize("bits", [8, 32])
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("name", list(OPT_ID))
def test_multi_call_equals_per_tensor_calls_and_the_reference(name, dtype, bits):
    code1, code2 = _codes()
    multi = _list(name, dtype, bits, seed=3)
    assert multi[MISALIGNED_P]["p"].data_ptr() % 16 and multi[MISALIGNED_S]["s1"].data_ptr() % 8
    single = _clone(multi)
    for rnd in range(2):
        _multi(name, dtype, bits, multi, code1, code2)
        _single(name, dtype, bits, single, code1, code2)
        torch.cuda.synchronize()
        nat.check()
        for i, (a, b) in enumerate(zip(multi, single)):
            _assert_bits_equal(a, b, f"{name} {dtype} {bits}-bit, round {rnd}, tensor {i}")
        for ts in (multi, single):
            for t in ts:
                t["step"] += 1
                t["g"].copy_((t["g"].float() * 0.7 - 0.02).to(t["g"].dtype))
    # the reference library on fresh, aligned copies (it is given no misaligned pointer)
    ref = _clone(_list(name, dtype, bits, seed=3), aligned=True)
    if not _reference(name, dtype, bits, ref, code1, code2):
        return
    got = _list(name, dtype, bits, seed=3)
    _multi(name, dtype, bits, got, code1, code2)
    torch.cuda.synchronize()
    nat.check()
    if bits == 8:  # the strictness of test_8bit_blockwise_update_equals_the_reference_cuda_library, over the list
        for k in ("s1", "s2"):
            if got[0][k] is None:
                continue
            o = np.concatenate([t[k].cpu().numpy() for t in got]).astype(np.int64)
            r = np.concatenate([t[k].cpu().numpy() for t in ref]).astype(np.int64)
            assert np.mean(o == r) > 0.999 and np.abs(o - r).max() <= 1, f"{name} {dtype}: {k} codes vs the reference"
    for i, (o, r) in enumerate(zip(got, ref)):
        what = f"{name} {dtype} {bits}-bit tensor {i} (n = {o['n']}) vs the reference library"
        if bits == 8:
            np.testing.assert_allclose(o["a1"].cpu().numpy(), r["a1"].cpu().numpy(), rtol=1e-6, atol=1e-12, err_msg=what)
            if o["a2"] is not None:
                np.testing.assert_allclose(o["a2"].cpu().numpy(), r["a2"].cpu().numpy(), rtol=1e-6, atol=1e-20, err_msg=what)
        else:
            _close(o["s1"].cpu().numpy(), r["s1"].cpu().numpy(), "fp32", what, ulps=4, atol=0, scale_ulps=4.0)
            if o["s2"] is not None:
                _close(o["s2"].cpu().numpy(), r["s2"].cpu().numpy(), "fp32", what, ulps=4, atol=0, scale_ulps=4.0)
        po, pr = o["p"].float().cpu().numpy(), r["p"].float().cpu().numpy()
        if bits == 8 and dtype != "fp32":
            assert np.array_equal(po, pr), f"{what}: 16-bit parameters differ"
        else:  # (32-bit state: an fma contracted differently here and there, as in test_gpu_optim.py)
            _close(po, pr, dtype, what, ulps=2.01, atol=0, scale_ulps=2.0)


@pytest.mark.parametrize("bits", [8, 32])
def test_a_list_longer_than_one_launch(bits):
    """2000 tiny tensors: several launches of at most optimizer_multi_capacity() descriptors, same results."""
    cap = optimizer_multi_capacity()
    assert 2000 > cap
    gen = torch.Generator(device="cpu").manual_seed(5)
    sizes = torch.randint(1, 700, (2000,), generator=gen).tolist()
    code1, code2 = _codes()
    ts = []
    for i, n in enumerate(sizes):
        nb = -(-n // 256)
        t = dict(p=torch.randn(n, generator=gen).to(torch.bfloat16).cuda(),
                 g=(torch.randn(n, generator=gen) * 0.1).to(torch.bfloat16).cuda(), n=n, step=1 + i % 9)
        if bits == 8:
            t.update(s1=torch.randint(0, 256, (n,), generator=gen, dtype=torch.uint8).cuda(),
                     s2=torch.randint(0, 256, (n,), generator=gen, dtype=torch.uint8).cuda(),
                     a1=(torch.rand(nb, generator=gen) * 0.05 + 1e-3).cuda(),
                     a2=(torch.rand(nb, generator=gen) * 0.002 + 1e-5).cuda())
        else:
            t.update(s1=(torch.rand(n, generator=gen) * 0.01).cuda(), s2=(torch.rand(n, generator=gen) * 0.001).cuda(),
                     a1=None, a2=None)
        ts.append(t)
    single = _clone(ts)
    _multi("adam", "bf16", bits, ts, code1, code2)
    _single("adam", "bf16", bits, single, code1, code2)
    torch.cuda.synchronize()
    nat.check()
    for i, (a, b) in enumerate(zip(ts, single)):
        _assert_bits_equal(a, b, f"adam {bits}-bit, tensor {i} of 2000")


def test_the_native_call_refuses_more_tensors_than_one_launch_takes():
    from bitsandbytes_b200 import cextension as cext

    cap = optimizer_multi_capacity()
    descs = (cext.OptimTensor * (cap + 1))()
    rc = nat.lib.cbnb_b200_optimizer_update_32bit_multi(0, 0, descs, cap + 1, 0.9, 0.999, 0.0, 0.0, 1e-8, 0.0, 1e-3, 1.0,
                                                        False, nat.stream())
    assert rc != 0
    with pytest.raises(RuntimeError, match="at most"):
        nat.check()


# ------------------------------------------------------------------------------------------ the optimizer classes
def _per_parameter(cls):
    """The optimizer with the per-parameter loop: a subclass that replaces update_step outside the package keeps one
    update_step call (and one single-tensor launch) per parameter."""

    class PerParameter(cls):
        def update_step(self, group, p, gindex, pindex):
            cls.update_step(self, group, p, gindex, pindex)

    return PerParameter


# name: (class, kwargs of both param groups' defaults)
CLASSES = {
    "Adam8bit": (lambda: bnb.optim.Adam8bit, dict(lr=1e-3)),
    "AdamW8bit": (lambda: bnb.optim.AdamW8bit, dict(lr=1e-3)),
    "PagedAdamW8bit": (lambda: bnb.optim.PagedAdamW8bit, dict(lr=1e-3)),
    "Lion8bit": (lambda: bnb.optim.Lion8bit, dict(lr=1e-4)),
    "AdEMAMix8bit": (lambda: bnb.optim.AdEMAMix8bit, dict(lr=1e-3, t_alpha=5, t_beta3=5)),
    "RMSprop8bit": (lambda: bnb.optim.RMSprop8bit, dict(lr=1e-3)),
    "Adagrad8bit": (lambda: bnb.optim.Adagrad8bit, dict(lr=1e-2)),
    "SGD8bit": (lambda: bnb.optim.SGD8bit, dict(lr=1e-2, momentum=0.9)),
    "Adam": (lambda: bnb.optim.Adam, dict(lr=1e-3)),
    "AdamW": (lambda: bnb.optim.AdamW, dict(lr=1e-3)),
    "PagedAdamW": (lambda: bnb.optim.PagedAdamW, dict(lr=1e-3)),
    "Lion": (lambda: bnb.optim.Lion, dict(lr=1e-4)),
    "AdEMAMix": (lambda: bnb.optim.AdEMAMix, dict(lr=1e-3, t_alpha=5, t_beta3=5)),
    "RMSprop": (lambda: bnb.optim.RMSprop, dict(lr=1e-3)),
    "Adagrad": (lambda: bnb.optim.Adagrad, dict(lr=1e-2)),
    "SGD": (lambda: bnb.optim.SGD, dict(lr=1e-2, momentum=0.9)),
}
# (shape, dtype): the min_8bit_size boundary (4095 / 4096), ragged and 16-bit parameters, one > 1e5 (paged state)
SHAPES = [((64, 64), torch.float32), ((4095,), torch.float32), ((4096,), torch.float32), ((33, 129), torch.bfloat16),
          ((300,), torch.bfloat16), ((128, 40), torch.bfloat16), ((7,), torch.float32), ((96, 256), torch.bfloat16),
          ((512, 256), torch.float32), ((1000,), torch.float32), ((24, 512), torch.float32), ((65,), torch.bfloat16),
          ((80, 64), torch.bfloat16), ((16, 256), torch.float32), ((400, 256), torch.bfloat16)]


def _params(name, seed):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    shapes = [(s, d) for s, d in SHAPES
              if not (name.startswith("AdEMAMix") and math.prod(s) >= 4096 and math.prod(s) % 256)]
    return [torch.nn.Parameter((torch.randn(s, generator=gen) * 0.1).to(d).cuda()) for s, d in shapes]


def _make(cls, params, kw):
    half = len(params) // 2
    kw2 = dict(kw, lr=kw["lr"] * 2, weight_decay=0.05)
    return cls([{"params": params[:half]}, {"params": params[half:], **kw2}], **kw)


def _states(opt, params):
    out = []
    for p in params:
        st = opt.state[p]
        out.append({k: v for k, v in st.items() if isinstance(v, torch.Tensor) and k not in ("qmap1", "qmap2")})
    return out


@pytest.mark.parametrize("name", list(CLASSES))
def test_grouped_step_equals_the_per_parameter_loop(name):
    get_cls, kw = CLASSES[name]
    cls = get_cls()
    mng = bnb.optim.GlobalOptimManager.get_instance()
    mng.initialize()
    try:
        pa, pb = _params(name, 1), _params(name, 1)
        big = next(i for i, p in enumerate(pa) if p.shape == (512, 256))
        for ps in (pa, pb):
            mng.override_config(ps[big], "optim_bits", 32)  # this weight keeps 32-bit state
        oa, ob = _make(cls, pa, kw), _make(_per_parameter(cls), pb, kw)
        assert oa._steps_in_groups() and not ob._steps_in_groups()
        gen = torch.Generator(device="cpu").manual_seed(2)
        for step in range(6):
            grads = [(torch.randn(p.shape, generator=gen) * 0.01).to(p.dtype).cuda() for p in pa]
            for i, (x, y, gr) in enumerate(zip(pa, pb, grads)):
                skip = (i + step) % 5 == 0  # some parameters have no gradient on some steps
                x.grad = None if skip else gr.clone()
                y.grad = None if skip else gr.clone()
            oa.step()
            ob.step()
            torch.cuda.synchronize()
            for i, (x, y) in enumerate(zip(pa, pb)):
                assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"{name} step {step}: parameter {i} differs"
            for i, (sa, sb) in enumerate(zip(_states(oa, pa), _states(ob, pb))):
                assert sa.keys() == sb.keys()
                for k in sa:
                    va, vb = sa[k].cuda(), sb[k].cuda()
                    assert torch.equal(va.view(torch.uint8), vb.view(torch.uint8)), f"{name} step {step}: {k} of {i}"
            if step == 2:  # a state_dict save / load in the middle of the run
                sda, sdb = oa.state_dict(), ob.state_dict()
                oa, ob = _make(cls, pa, kw), _make(_per_parameter(cls), pb, kw)
                oa.load_state_dict(sda)
                ob.load_state_dict(sdb)
        kinds = [oa.state[p]["state1"].dtype for p in (pa[1], pa[2], pa[big])]  # 4095, 4096 elements; the override
        want = [torch.float32, torch.uint8, torch.float32] if name.endswith("8bit") else [torch.float32] * 3
        assert kinds == want
    finally:
        mng.initialize()


# ------------------------------------------------------------------------------------------ launches per step
def lora_shapes(r):
    """LoRA A / B on all seven projections of the 32 layers of a Llama-3-8B (hidden 4096, 8 KV heads of 128,
    intermediate 14336): 448 tensors."""
    proj = [(4096, 4096), (4096, 1024), (4096, 1024), (4096, 4096), (4096, 14336), (4096, 14336), (14336, 4096)]
    return [s for _ in range(32) for i, o in proj for s in ((r, i), (o, r))]


def test_one_adamw8bit_step_over_the_lora_set_launches_one_kernel_per_capacity_chunk():
    from torch.profiler import ProfilerActivity, profile, record_function

    gen = torch.Generator(device="cuda").manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(s, device="cuda", generator=gen, dtype=torch.bfloat16) * 0.02)
              for s in lora_shapes(16)]
    assert len(params) == 448
    for p in params:
        p.grad = torch.randn(p.shape, device="cuda", generator=gen, dtype=p.dtype) * 1e-3
    opt = bnb.optim.AdamW8bit(params, lr=1e-4)
    opt.step()  # (the first step also creates the state)
    opt2 = bnb.optim.AdamW8bit(params, lr=1e-4)
    opt2.load_state_dict(opt.state_dict())
    assert len({id(opt2.state[p]["qmap1"]) for p in params}) == 1, "the reloaded code books are shared again"
    torch.cuda.synchronize()
    # one profiler session; a step's kernels are those that start inside its range (which ends in a synchronise)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)  # (the first kernels of a session can go unrecorded)
        torch.cuda.synchronize()
        for name, o in (("step", opt), ("step after load_state_dict", opt2)):
            with record_function(name):
                o.step()
                torch.cuda.synchronize()
    events = prof.events()
    kernels = [e for e in events if e.device_type == torch.autograd.DeviceType.CUDA and "optim" in e.name]
    want = math.ceil(len(params) / optimizer_multi_capacity())
    for name in ("step", "step after load_state_dict"):
        r = next(e.time_range for e in events if e.name == name)
        mine = [e.name for e in kernels if r.start <= e.time_range.start <= r.end]
        assert len(mine) == want and all("optim8_2state_kernel" in n for n in mine), (name, mine)
    assert len(kernels) == 2 * want
