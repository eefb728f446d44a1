"""GPU tests of global gradient-norm clipping for the data-parallel step (``ShardedOptimizer.clip_grad_norm_``,
csrc/optim.cu ``peer_norm_kernel`` / ``clip_coef_kernel`` and the ``_peers_scaled`` entries).

* The norm entry, with w = 1..8 "ranks" simulated as separate buffers passed as raw addresses, against the float64
  oracle of the reduced gradient T(rank-order fp32 sum * grad_scale): L2 within one fp32 ulp, inf exactly; fp32, fp16
  and bf16; partial blocks, pieces under one block, several chunks, misaligned buffers, more pieces than one launch
  holds; zeros, NaN and Inf; the same bits on a second run.
* The coefficient's bits against torch's ``(max_norm / (total_norm + 1e-6)).clamp(max=1.0)``.
* The scaled peer entries against the multi-tensor entries on the reduced gradient with ``gnorm_scale = coefficient``,
  bit for bit (fp32 32-bit Lion: within the bounds of test_gpu_sharded_optim); with a NULL coefficient, the unscaled
  peer entries' bits; rejected arguments write nothing.
* ``clip_grad_norm_`` at one rank makes no host synchronisation.
* In one process per GPU (torch.distributed.run, 1 and 2 processes): training with clipping that sometimes clips,
  against an unsharded optimizer fed the reduced gradient with gnorm_scale set to the returned coefficient.
"""
import ctypes as ct
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.functional as F
from bitsandbytes_b200 import cextension as cext
from bitsandbytes_b200.backends import cuda as backend
from bitsandbytes_b200.backends.cuda import (optimizer_clip_coef, optimizer_grad_norm_peers,
                                             optimizer_update_32bit_multi_peers,
                                             optimizer_update_8bit_blockwise_multi_peers)
from tests import _native as nat
from tests.test_gpu_sharded_optim import _DT, _OPTS, _PIECES, _bits, _case, _lion_fp32_bounds, _ref_grad

pytestmark = pytest.mark.gpu


def _finite_case(dtype, w, shift, seed, name="adam", eight=True):
    """_case's buffers with its NaN / Inf gradients replaced by finite values."""
    offs, numel, grads, g_local, p_local, states = _case(name, dtype, eight, w, shift, seed)
    for g in grads:
        torch.nan_to_num_(g, nan=0.5, posinf=3.0, neginf=-3.0)
    return offs, numel, grads, g_local, p_local, states


def _norm(pieces, grads, g_local, scale, norm_type, max_norm=1.0):
    """(accumulated fp64 value, total norm, coefficient) through the two entries, one simulated rank."""
    acc = torch.zeros(1, dtype=torch.float64, device="cuda")
    optimizer_grad_norm_peers(pieces, [g.data_ptr() for g in grads], g_local, scale, norm_type, acc)
    out = torch.empty(2, dtype=torch.float32, device="cuda")
    optimizer_clip_coef(acc, norm_type, max_norm, out)
    torch.cuda.synchronize()
    return acc, out[0], out[1]


def _oracle(grads, scale, dtype, spans, norm_type):
    red = _ref_grad(grads, scale, dtype).double()
    vals = torch.cat([red[o:o + n] for o, n in spans])
    return vals.abs().max().item() if norm_type == math.inf else vals.square().sum().sqrt().item()


def _within_one_ulp(got, want):
    w32 = np.float32(want)
    return abs(float(got) - want) <= float(np.spacing(np.abs(w32)))


def _torch_coef(norm, max_norm):
    return (max_norm / (norm.reshape(1).clone() + 1e-6)).clamp(max=1.0)[0]


@pytest.mark.parametrize("shift", [0, 1])
@pytest.mark.parametrize("norm_type", [2.0, math.inf])
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("w", range(1, 9))
def test_norm_matches_float64_oracle(w, dtype, norm_type, shift):
    td = _DT[dtype]
    scale = 1.0 / 3.0
    offs, numel, grads, g_local, _, _ = _finite_case(td, w, shift, seed=w * 11 + shift)
    pieces = [g_local[o:o + n] for o, n in zip(offs, _PIECES)]
    acc, norm, coef = _norm(pieces, grads, g_local, scale, norm_type, max_norm=0.25)
    want = _oracle(grads, scale, td, list(zip(offs, _PIECES)), norm_type)
    if norm_type == math.inf:
        assert float(norm) == np.float32(want) and acc.item() == want
    else:
        assert _within_one_ulp(norm, want), (float(norm), want)
        assert abs(acc.item() - want * want) <= 1e-12 * want * want
    assert torch.equal(_bits(coef), _bits(_torch_coef(norm, 0.25)))
    acc2, norm2, coef2 = _norm(pieces, grads, g_local, scale, norm_type, max_norm=0.25)  # deterministic
    assert torch.equal(acc2.view(torch.int64), acc.view(torch.int64)) and torch.equal(_bits(norm2), _bits(norm))


@pytest.mark.parametrize("norm_type", [2.0, math.inf])
def test_more_pieces_than_one_launch_holds(norm_type):
    cap = backend.optimizer_peers_capacity()
    k, w, td = cap * 2 + 17, 3, torch.bfloat16
    numel = k * 256
    gen = torch.Generator().manual_seed(5)
    grads = [(torch.randn(numel, generator=gen) * 4).to(td).cuda() for _ in range(w)]
    spans = [(256 * i, 1 + (i * 37) % 256) for i in range(k)]
    pieces = [grads[0][o:o + n] for o, n in spans]
    _, norm, _ = _norm(pieces, grads, grads[0], 0.5, norm_type)
    want = _oracle(grads, 0.5, td, spans, norm_type)
    assert float(norm) == np.float32(want) if norm_type == math.inf else _within_one_ulp(norm, want)


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_zero_nan_inf_gradients(dtype):
    td = _DT[dtype]
    offs, numel, grads, g_local, _, _ = _finite_case(td, 2, 0, seed=3)
    pieces = [g_local[o:o + n] for o, n in zip(offs, _PIECES)]
    srcs = grads
    for g in grads:
        g.zero_()
    for nt in (2.0, math.inf):
        acc, norm, coef = _norm(pieces, srcs, g_local, 1.0, nt, max_norm=1.0)
        assert acc.item() == 0.0 and float(norm) == 0.0 and float(coef) == 1.0
    grads[1][offs[3] + 100] = float("inf")
    for nt in (2.0, math.inf):
        _, norm, coef = _norm(pieces, srcs, g_local, 1.0, nt)
        assert math.isinf(float(norm)) and float(coef) == 0.0
        assert torch.equal(_bits(coef), _bits(_torch_coef(norm, 1.0)))
    grads[0][offs[1] + 2] = float("nan")
    for nt in (2.0, math.inf):
        _, norm, coef = _norm(pieces, srcs, g_local, 1.0, nt)
        assert math.isnan(float(norm)) and math.isnan(float(coef))


def test_coefficient_bits_equal_torch():
    """Rank-order fp64 sums, sqrt rounded once, and torch's coefficient over many norms and max_norm values."""
    gen = torch.Generator().manual_seed(0)
    for w in (1, 2, 5, 8):
        for trial in range(60):
            v = (torch.rand(w, generator=gen, dtype=torch.float64) * 10.0 ** torch.randint(-12, 12, (1,),
                                                                                           generator=gen)).cuda()
            max_norm = float(torch.rand(1, generator=gen)) * 10.0 ** int(torch.randint(-4, 4, (1,), generator=gen))
            for nt in (2.0, math.inf):
                out = torch.empty(2, dtype=torch.float32, device="cuda")
                optimizer_clip_coef(v, nt, max_norm, out)
                vals = v.tolist()
                t = vals[0]
                for x in vals[1:]:
                    t = max(t, x) if nt == math.inf else t + x
                assert float(out[0]) == float(np.float32(t if nt == math.inf else math.sqrt(t)))
                assert torch.equal(_bits(out[1]), _bits(_torch_coef(out[0], max_norm))), (vals, max_norm)


def _scaled_run(name, td, eight, offs, g_local, p_local, states, srcs, dsts, scale, coef):
    """One update through the scaled entries; coef: a one-element CUDA tensor, or 0 for a NULL pointer."""
    b1, b2 = _OPTS[name]
    g = [g_local[o:o + n] for o, n in zip(offs, _PIECES)]
    p = [p_local[o:o + n] for o, n in zip(offs, _PIECES)]
    s1 = [st["state1"] for st in states]
    s2 = [st["state2"] for st in states] if name == "adam" else None
    steps = [3 + i for i in range(len(_PIECES))]
    lr, eps, wd = 1e-3, 1e-8, 0.01
    q1, q2 = F.create_dynamic_map(signed=True).cuda(), F.create_dynamic_map(signed=False).cuda()
    if not isinstance(coef, int):
        if eight:
            optimizer_update_8bit_blockwise_multi_peers(name, g, p, s1, s2, b1, b2, 0.0, 0.0, eps, steps, lr, q1, q2,
                                                        [st["absmax1"] for st in states],
                                                        [st["absmax2"] for st in states] if s2 else None, wd, srcs,
                                                        dsts, g_local, p_local, scale, gnorm_scale_dev=coef)
        else:
            optimizer_update_32bit_multi_peers(name, g, p, s1, s2, b1, b2, 0.0, 0.0, eps, wd, steps, lr, srcs, dsts,
                                               g_local, p_local, scale, gnorm_scale_dev=coef)
        return
    # the NULL pointer: straight through the C entry
    what = "test"
    a1 = [st["absmax1"] for st in states] if eight else None
    a2 = [st["absmax2"] for st in states] if eight and s2 else None
    g0, descs, _ = backend._optimizer_list(what, name, backend._OPTIMIZER_ID, g, p, s1, s2, a1, a2, steps, eight)
    sp, dp = backend._peer_args(what, g, p, steps, srcs, dsts, g_local, p_local)
    if eight:
        fn = nat.lib.cbnb_b200_optimizer_update_8bit_blockwise_multi_peers_scaled
        scalars = (b1, b2, 0.0, 0.0, eps, wd, lr, q1.data_ptr(), q2.data_ptr() if s2 else None, False, None)
    else:
        fn = nat.lib.cbnb_b200_optimizer_update_32bit_multi_peers_scaled
        scalars = (b1, b2, 0.0, 0.0, eps, wd, lr, False, None)
    backend._launch_peers(what, fn, name, g0, descs, sp, dp, g_local, p_local, scale, scalars)


def _multi_ref(name, eight, offs, g_ref, p_ref, states, gnorm_scale):
    b1, b2 = _OPTS[name]
    g = [g_ref[o:o + n] for o, n in zip(offs, _PIECES)]
    p = [p_ref[o:o + n] for o, n in zip(offs, _PIECES)]
    s1 = [st["state1"] for st in states]
    s2 = [st["state2"] for st in states] if name == "adam" else None
    steps = [3 + i for i in range(len(_PIECES))]
    lr, eps, wd = 1e-3, 1e-8, 0.01
    if eight:
        q1, q2 = F.create_dynamic_map(signed=True).cuda(), F.create_dynamic_map(signed=False).cuda()
        F.optimizer_update_8bit_blockwise_multi(name, g, p, s1, s2, b1, b2, 0.0, 0.0, eps, steps, lr, q1, q2,
                                                [st["absmax1"] for st in states],
                                                [st["absmax2"] for st in states] if s2 else None, wd,
                                                gnorm_scale=gnorm_scale)
    else:
        F.optimizer_update_32bit_multi(name, g, p, s1, b1, eps, steps, lr, s2, b2, 0.0, 0.0, wd, gnorm_scale)


def _scaled_check(name, dtype, eight, w, shift, null):
    td = _DT[dtype]
    scale = 1.0 / 3.0
    offs, numel, grads, g_local, p_local, states = _finite_case(td, w, shift, seed=w * 5 + shift + 1, name=name,
                                                                eight=eight)
    pieces = [g_local[o:o + n] for o, n in zip(offs, _PIECES)]
    _, norm, _ = _norm(pieces, grads, g_local, scale, 2.0)
    out = torch.empty(2, dtype=torch.float32, device="cuda")
    acc = torch.zeros(1, dtype=torch.float64, device="cuda")
    optimizer_grad_norm_peers(pieces, [g.data_ptr() for g in grads], g_local, scale, 2.0, acc)
    optimizer_clip_coef(acc, 2.0, float(norm) / 3.0, out)        # a coefficient that clips, about 1/3
    coef = out[1:]
    gscale = 1.0 if null else float(coef)
    assert null or 0.3 < gscale < 0.4
    ref_states = [{k: v.clone() for k, v in st.items()} for st in states]
    states0 = [st["state1"].clone() for st in states]
    g_ref = torch.empty(numel + shift, dtype=td, device="cuda")[shift:]
    g_ref.copy_(_ref_grad(grads, scale, td))
    p_ref = torch.empty(numel + shift, dtype=td, device="cuda")[shift:]
    p_ref.copy_(p_local)
    p_before = p_local.clone()
    dsts = [torch.full((numel + shift,), float("nan"), dtype=td, device="cuda")[shift:] for _ in range(w)]
    _scaled_run(name, td, eight, offs, g_local, p_local, states, [g.data_ptr() for g in grads],
                [d.data_ptr() for d in dsts], scale, 0 if null else coef)
    _multi_ref(name, eight, offs, g_ref, p_ref, ref_states, gscale)
    torch.cuda.synchronize()
    owned = torch.zeros(numel, dtype=torch.bool, device="cuda")
    for o, n in zip(offs, _PIECES):
        owned[o:o + n] = True
    loose = name == "lion" and not eight and td == torch.float32
    g_scaled = (g_ref.float() * gscale).to(td) if loose else None
    for d in dsts:
        if loose:
            _lion_fp32_bounds(offs, g_scaled, p_before, states0, d, p_ref, states, ref_states)
        else:
            assert torch.equal(_bits(d[owned]), _bits(p_ref[owned])), "parameters"
        assert torch.isnan(d[~owned]).all(), "a write outside the pieces"
    assert torch.equal(_bits(p_local), _bits(p_before))
    if not loose:
        for st, rs in zip(states, ref_states):
            for k in st:
                assert torch.equal(_bits(st[k]), _bits(rs[k])), k


@pytest.mark.parametrize("w", [1, 2, 5, 8])
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("eight", [True, False])
@pytest.mark.parametrize("name", list(_OPTS))
def test_scaled_entries_equal_multi_with_gnorm_scale(name, eight, dtype, w):
    _scaled_check(name, dtype, eight, w, shift=0, null=False)


@pytest.mark.parametrize("w", [1, 3])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("eight", [True, False])
@pytest.mark.parametrize("name", ["adam", "momentum"])
def test_scaled_entries_misaligned_and_null(name, eight, dtype, w):
    _scaled_check(name, dtype, eight, w, shift=1, null=False)
    _scaled_check(name, dtype, eight, w, shift=0, null=True)


def test_rejected_arguments_write_nothing():
    td = torch.bfloat16
    offs, numel, grads, g_local, p_local, states = _finite_case(td, 2, 0, seed=1)
    acc = torch.full((1,), 7.0, dtype=torch.float64, device="cuda")
    d = cext.OptimTensor(0, g_local[offs[0]:].data_ptr(), 0, 0, 0, 0, _PIECES[0], 0, 0)
    stream = torch.cuda.current_stream().cuda_stream

    def norm(dtype=2, count=1, srcs=None, world=2, gl=None, numel_=numel, acc_=None):
        srcs = [g.data_ptr() for g in grads] if srcs is None else srcs
        a = (ct.c_void_p * max(1, len(srcs)))(*srcs)
        rc = nat.lib.cbnb_b200_optimizer_grad_norm_peers(dtype, ct.addressof(d), count, ct.cast(a, ct.c_void_p), world,
                                                         g_local.data_ptr() if gl is None else gl, numel_, 1.0, False,
                                                         acc.data_ptr() if acc_ is None else acc_, stream)
        torch.cuda.synchronize()
        return rc

    for kw in [dict(count=-1), dict(count=10_000), dict(dtype=3)]:
        assert norm(**kw) == 100, kw
        with pytest.raises(RuntimeError, match="norm"):
            nat.check()
    for kw in [dict(world=0), dict(world=9), dict(srcs=[grads[0].data_ptr(), 0]), dict(gl=0),
               dict(gl=g_local.data_ptr() + 1), dict(numel_=offs[0] + _PIECES[0] - 1), dict(acc_=0),
               dict(acc_=acc.data_ptr() + 4), dict(gl=g_local[offs[0] + 2:].data_ptr())]:
        assert norm(**kw) == 1, kw
        with pytest.raises(RuntimeError, match="norm"):
            nat.check()
    assert acc.item() == 7.0
    out = torch.full((2,), float("nan"), device="cuda")
    for vals, world, o in [(acc.data_ptr(), 0, out.data_ptr()), (0, 1, out.data_ptr()), (acc.data_ptr(), 1, 0),
                           (acc.data_ptr(), 1, out.data_ptr() + 2)]:
        assert nat.lib.cbnb_b200_optimizer_clip_coef(vals, world, False, 1.0, o, stream) == 1
        with pytest.raises(RuntimeError, match="clip_coef"):
            nat.check()
    torch.cuda.synchronize()
    assert torch.isnan(out).all()
    assert norm() == 0
    nat.check()
    with pytest.raises(ValueError):
        optimizer_grad_norm_peers([g_local[offs[0]:offs[0] + 5]], [grads[0].data_ptr()], g_local, 1.0, 1.0, acc)
    with pytest.raises(ValueError):
        optimizer_clip_coef(acc, 3, 1.0, torch.empty(2, device="cuda"))
    # the scaled update: a bad peer argument returns 1 and writes nothing
    dst = torch.full((numel,), float("nan"), dtype=td, device="cuda")
    s1_before = states[0]["state1"].clone()
    coef = torch.full((1,), 0.5, device="cuda")
    q1, q2 = F.create_dynamic_map(signed=True).cuda(), F.create_dynamic_map(signed=False).cuda()
    u = cext.OptimTensor(p_local[offs[0]:].data_ptr(), g_local[offs[0]:].data_ptr(), states[0]["state1"].data_ptr(),
                         states[0]["state2"].data_ptr(), states[0]["absmax1"].data_ptr(),
                         states[0]["absmax2"].data_ptr(), _PIECES[0], 1, 0)
    srcs = (ct.c_void_p * 2)(*[g.data_ptr() for g in grads])
    dsts = (ct.c_void_p * 1)(dst.data_ptr())
    for world, ndst, rc_want in [(0, 1, 1), (2, 0, 1), (9, 1, 1)]:
        rc = nat.lib.cbnb_b200_optimizer_update_8bit_blockwise_multi_peers_scaled(
            0, 2, ct.addressof(u), 1, ct.cast(srcs, ct.c_void_p), world, ct.cast(dsts, ct.c_void_p), ndst,
            g_local.data_ptr(), p_local.data_ptr(), numel, 0.5, 0.9, 0.999, 0.0, 0.0, 1e-8, 0.0, 1e-3, q1.data_ptr(),
            q2.data_ptr(), False, coef.data_ptr(), stream)
        assert rc == rc_want
        with pytest.raises(RuntimeError, match="scaled"):
            nat.check()
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.equal(states[0]["state1"], s1_before)
    with pytest.raises(ValueError, match="gnorm_scale_dev"):
        optimizer_update_8bit_blockwise_multi_peers(
            "adam", [g_local[offs[0]:offs[0] + _PIECES[0]]], [p_local[offs[0]:offs[0] + _PIECES[0]]],
            [states[0]["state1"]], [states[0]["state2"]], 0.9, 0.999, 0.0, 0.0, 1e-8, [1], 1e-3, q1, q2,
            [states[0]["absmax1"]], [states[0]["absmax2"]], 0.0, [grads[0].data_ptr()], [dst.data_ptr()], g_local,
            p_local, 0.5, gnorm_scale_dev=torch.ones(1, dtype=torch.float64, device="cuda"))


def test_one_rank_clip_makes_no_host_sync():
    torch.manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(s, device="cuda").to(dt)) for s, dt in
              [((300, 40), torch.bfloat16), ((77,), torch.bfloat16), ((5000,), torch.float32)]]
    opt = bnb.optim.ShardedOptimizer(bnb.optim.AdamW8bit(params, lr=1e-3, min_8bit_size=4096))
    for p in params:
        p.grad.copy_(torch.randn_like(p))
    want = math.sqrt(sum(p.grad.double().square().sum().item() for p in params))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        total = opt.clip_grad_norm_(1.0)
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _within_one_ulp(total, want)


# ------------------------------------------------------------------------------------------ processes
_SCRIPT = r"""
import math, os, sys, torch, numpy as np, torch.distributed as dist
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import bitsandbytes_b200 as bnb
import bitsandbytes_b200.optim.optimizer as bopt

rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
F = bopt.F


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


class Scaled:
    # the unsharded optimizer's launches with gnorm_scale set to the clip coefficient
    def __init__(self, coef):
        self.coef, self.calls = coef, 0

    def __getattr__(self, name):
        return getattr(F, name)

    def _pos(self, fn, a, kw):
        self.calls += 1
        a = list(a)
        a[13] = self.coef
        return fn(*a, **kw)

    def _kw(self, fn, a, kw):
        self.calls += 1
        kw["gnorm_scale"] = self.coef
        return fn(*a, **kw)

    def optimizer_update_32bit_multi(self, *a, **kw):
        return self._pos(F.optimizer_update_32bit_multi, a, kw)

    def optimizer_update_32bit(self, *a, **kw):
        return self._pos(F.optimizer_update_32bit, a, kw)

    def optimizer_update_8bit_blockwise_multi(self, *a, **kw):
        return self._kw(F.optimizer_update_8bit_blockwise_multi, a, kw)

    def optimizer_update_8bit_blockwise(self, *a, **kw):
        return self._kw(F.optimizer_update_8bit_blockwise, a, kw)


class Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(256, 384).to(torch.bfloat16)      # 8-bit weight, 32-bit bias
        self.b = torch.nn.Linear(384, 300).to(torch.bfloat16)
        self.n = torch.nn.LayerNorm(300)                           # fp32, 32-bit state
        self.c = torch.nn.Linear(300, 5000, bias=False)            # fp32, 8-bit

    def forward(self, x):
        h = self.b(torch.relu(self.a(x.to(torch.bfloat16))))
        return self.c(self.n(h.float()))


def reduced(t, scale):
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous())
    acc = parts[0].float()
    for q in parts[1:]:
        acc = acc + q.float()
    return (acc * torch.tensor(scale, dtype=torch.float32, device=dev)).to(t.dtype)


MAKERS = {"AdamW8bit": lambda p: bnb.optim.AdamW8bit(p, lr=1e-3, weight_decay=0.01, min_8bit_size=4096),
          "Lion8bit": lambda p: bnb.optim.Lion8bit(p, lr=1e-4, min_8bit_size=4096),
          "Adam32bit": lambda p: bnb.optim.Adam32bit(p, lr=1e-3)}
clipped = unclipped = 0
for kind, make in MAKERS.items():
    for nt in (2.0, math.inf):
        torch.manual_seed(0)
        model = Net().to(dev)
        torch.manual_seed(0)
        ref = Net().to(dev)
        opt = bnb.optim.ShardedOptimizer(make(model.parameters()))
        ref_opt = make(ref.parameters())
        norms = []
        for step in range(5):
            g = torch.Generator().manual_seed(100 * step + rank)
            x, y = torch.randn(16, 256, generator=g).to(dev), torch.randn(16, 5000, generator=g).to(dev)
            torch.nn.functional.mse_loss(model(x), y).backward()
            reds = [reduced(p.grad, opt.grad_scale) for p in model.parameters()]
            want = max(r.double().abs().max().item() for r in reds) if nt == math.inf else \
                math.sqrt(sum(r.double().square().sum().item() for r in reds))
            # max_norm near the norm, so that some steps clip and some do not
            max_norm = want * (0.7 if step % 2 == 0 else 1.3)
            max_norm = float(torch.tensor(max_norm, dtype=torch.float32))
            every = [torch.empty(1, device=dev) for _ in range(world)]
            dist.all_gather(every, torch.tensor([max_norm], device=dev))
            max_norm = float(every[0])                              # rank 0's value on every rank
            total = opt.clip_grad_norm_(max_norm, norm_type=nt)
            coef = float((max_norm / (total.reshape(1).clone() + 1e-6)).clamp(max=1.0))
            tb = bits(total.reshape(1).clone())
            allb = [torch.empty_like(tb) for _ in range(world)]
            dist.all_gather(allb, tb)
            assert all(torch.equal(b, tb) for b in allb), f"rank {rank}: the norm differs across ranks"
            if nt == math.inf:
                assert float(total) == float(np.float32(want)), (float(total), want)
            else:
                assert abs(float(total) - want) <= float(np.spacing(np.float32(want))), (float(total), want)
            clipped += coef < 1.0
            unclipped += coef == 1.0
            for q, r in zip(ref.parameters(), reds):
                q.grad = r
            bopt.F = Scaled(coef)
            try:
                ref_opt.step()
                assert bopt.F.calls > 0
            finally:
                bopt.F = F
            ref_opt.zero_grad()
            opt.step()
            opt.zero_grad()
            for (name, p), q in zip(model.named_parameters(), ref.parameters()):
                assert torch.equal(bits(p.detach()), bits(q.detach())), f"rank {rank}: {kind} {nt} step {step} {name}"
assert clipped and unclipped, (clipped, unclipped)
dist.barrier()
dist.destroy_process_group()
print("CLIP_OK", rank)
"""


@pytest.mark.parametrize("nproc", [1, 2])
def test_processes_clipped_training_equals_unsharded(tmp_path, nproc):
    """One process per GPU: AdamW8bit, Lion8bit and Adam32bit over bf16 and fp32 tensors train five steps with
    clip_grad_norm_ (L2 and inf), max_norm alternately below and above the norm; the norm has the same bits on every
    rank and matches the float64 oracle of the all-gathered reduced gradient; the parameters equal, bit for bit, an
    unsharded optimizer's fed the reduced gradient with gnorm_scale = the coefficient, after every step."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "clip.py"
    script.write_text(_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29691 + nproc), str(script)],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and r.stdout.count("CLIP_OK") == nproc, r.stdout[-3000:] + r.stderr[-4000:]
