"""GPU tests of the data-parallel optimizer step (``bnb.optim.ShardedOptimizer``, csrc/optim.cu peer instances).

* The two C entries, with w = 1..8 "ranks" simulated as separate buffers passed as raw addresses, against the
  multi-tensor update fed the rank-order fp32 sum of the ranks' gradients times grad_scale, rounded once: parameters
  in every destination and the states bit for bit, for every supported optimizer, dtype and state width, with partial
  last blocks, misaligned buffers (element path), NaN / Inf gradients and grad_scale 1/3 and 1; nothing is written
  outside the pieces (NaN canaries), and rejected arguments return codes with nothing written.
* In one process per GPU (torch.distributed.run, 1 and 2 processes): a small model with 8-bit and 32-bit tensors of two
  dtypes, gradient accumulation and an LR scheduler, against an unsharded optimizer on each rank fed the all-gathered,
  rank-order-reduced gradient; every rank's parameters; the consolidated checkpoint (gathered to rank 0) loaded into a
  plain optimizer and back into a sharded one, training on with equal bits.
"""
import ctypes as ct
import os
import subprocess
import sys

import pytest
import torch

import bitsandbytes_b200.functional as F
from bitsandbytes_b200 import cextension as cext
from bitsandbytes_b200.backends.cuda import (optimizer_update_32bit_multi_peers,
                                             optimizer_update_8bit_blockwise_multi_peers)
from tests import _native as nat

pytestmark = pytest.mark.gpu

_DT = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}
# name -> (beta1, beta2)
_OPTS = {"adam": (0.9, 0.999), "momentum": (0.9, 0.0), "rmsprop": (0.9, 0.0), "adagrad": (0.0, 0.0),
         "lion": (0.9, 0.99)}
# piece sizes: whole blocks, a partial last block, less than a block, several chunks of the 32-bit kernel
_PIECES = [1024, 300, 7, 4096 + 256 * 3 + 5, 256]


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


def _ref_grad(grads, scale, dtype):
    acc = grads[0].float()
    for g in grads[1:]:
        acc = acc + g.float()
    return (acc * torch.tensor(scale, dtype=torch.float32, device=acc.device)).to(dtype)


def _case(name, dtype, eight, w, shift, seed):
    """Flat buffers of the local rank (gradient, parameters) and w gradient copies, pieces at block-aligned offsets,
    states of mid-training values.  shift > 0 moves every buffer `shift` elements off 16-byte alignment."""
    gen = torch.Generator().manual_seed(seed)
    offs, o = [], 256
    for n in _PIECES:
        offs.append(o)
        o += -(-n // 256) * 256 + 256
    numel = o

    def buf(fill):
        b = fill(numel + shift)
        return b[shift:]

    grads = []
    for r in range(w):
        g = (torch.randn(numel, generator=gen) * 2.0 ** torch.randint(-8, 4, (numel,), generator=gen)).to(dtype)
        if r == min(1, w - 1):
            g[offs[0] + 3] = float("nan")
            g[offs[3] + 100] = float("inf")
            g[offs[3] + 101] = -float("inf")
        grads.append(buf(lambda m: torch.zeros(m, dtype=dtype, device="cuda")))
        grads[-1].copy_(g)
    p_local = buf(lambda m: torch.zeros(m, dtype=dtype, device="cuda"))
    p_local.copy_((torch.randn(numel, generator=gen) * 0.5).to(dtype))
    g_local = grads[0]
    two = name == "adam"
    states = []
    for n in _PIECES:
        st = {}
        if eight:
            nb = -(-n // 256)
            lo = 128 if name in ("rmsprop", "adagrad") else 0
            st["state1"] = torch.randint(lo, 256, (n,), generator=gen, dtype=torch.uint8).cuda()
            st["absmax1"] = (torch.rand(nb, generator=gen) * 0.05 + 1e-3).cuda()
            if two:
                st["state2"] = torch.randint(0, 256, (n,), generator=gen, dtype=torch.uint8).cuda()
                st["absmax2"] = (torch.rand(nb, generator=gen) * 0.01 + 1e-4).cuda()
        else:
            st["state1"] = (torch.randn(n, generator=gen) * 0.01).cuda()
            if name in ("rmsprop", "adagrad"):
                st["state1"] = st["state1"].abs()
            if two:
                st["state2"] = (torch.rand(n, generator=gen) * 1e-4).cuda()
        states.append(st)
    return offs, numel, grads, g_local, p_local, states


def _run(name, dtype, eight, offs, grads, g_local, p_local, states, srcs, dsts, scale, peers=True, g_ref=None,
         p_ref=None):
    """One update of the pieces: through the peer entry (peers=True) or the existing multi-tensor one on g_ref."""
    b1, b2 = _OPTS[name]
    g = [(g_local if peers else g_ref)[o:o + n] for o, n in zip(offs, _PIECES)]
    p = [(p_local if peers else p_ref)[o:o + n] for o, n in zip(offs, _PIECES)]
    s1 = [st["state1"] for st in states]
    s2 = [st["state2"] for st in states] if name == "adam" else None
    steps = [3 + i for i in range(len(_PIECES))]
    lr, eps, wd = 1e-3, 1e-8, 0.01
    if eight:
        q1, q2 = F.create_dynamic_map(signed=True).cuda(), F.create_dynamic_map(signed=False).cuda()
        a1 = [st["absmax1"] for st in states]
        a2 = [st["absmax2"] for st in states] if name == "adam" else None
        if peers:
            optimizer_update_8bit_blockwise_multi_peers(name, g, p, s1, s2, b1, b2, 0.0, 0.0, eps, steps, lr, q1, q2,
                                                        a1, a2, wd, srcs, dsts, g_local, p_local, scale)
        else:
            F.optimizer_update_8bit_blockwise_multi(name, g, p, s1, s2, b1, b2, 0.0, 0.0, eps, steps, lr, q1, q2, a1,
                                                    a2, wd)
    elif peers:
        optimizer_update_32bit_multi_peers(name, g, p, s1, s2, b1, b2, 0.0, 0.0, eps, wd, steps, lr, srcs, dsts,
                                           g_local, p_local, scale)
    else:
        F.optimizer_update_32bit_multi(name, g, p, s1, b1, eps, steps, lr, s2, b2, 0.0, 0.0, wd)


def _check(name, dtype, eight, w, shift, scale):
    td = _DT[dtype]
    offs, numel, grads, g_local, p_local, states = _case(name, td, eight, w, shift, seed=w * 7 + shift)
    ref_states = [{k: v.clone() for k, v in st.items()} for st in states]
    states0 = [st["state1"].clone() for st in states]
    # the reference's buffers have the same alignment, so that it takes the same (vector or element) path
    g_ref = torch.empty(numel + shift, dtype=td, device="cuda")[shift:]
    g_ref.copy_(_ref_grad(grads, scale, td))
    p_ref = torch.empty(numel + shift, dtype=td, device="cuda")[shift:]
    p_ref.copy_(p_local)
    p_before = p_local.clone()
    dsts = []
    for _ in range(w):
        d = torch.full((numel + shift,), float("nan"), dtype=td, device="cuda")[shift:]
        dsts.append(d)
    _run(name, td, eight, offs, grads, g_local, p_local, states, [t.data_ptr() for t in grads],
         [t.data_ptr() for t in dsts], scale)
    _run(name, td, eight, offs, None, None, None, ref_states, None, None, scale, peers=False, g_ref=g_ref, p_ref=p_ref)
    torch.cuda.synchronize()
    owned = torch.zeros(numel, dtype=torch.bool, device="cuda")
    for o, n in zip(offs, _PIECES):
        owned[o:o + n] = True
    # fp32 parameters with 32-bit Lion state: the multi-tensor kernel contracts the decoupled weight decay and the step,
    # and the products of sign(beta1 * m + (1 - beta1) * g), into one fma in some unrolled copies of its element loop
    # and not in others, with no rounding to a 16-bit dtype to hide it, so its own result depends on the element's place
    # in the loop.  There each value is bounded by what one contraction can change (_lion_fp32_bounds); every other
    # combination is bit for bit.
    loose = name == "lion" and not eight and td == torch.float32
    for d in dsts:
        if loose:
            _lion_fp32_bounds(offs, g_ref, p_before, states0, d, p_ref, states, ref_states)
        else:
            assert torch.equal(_bits(d[owned]), _bits(p_ref[owned])), "parameters"
        assert torch.isnan(d[~owned]).all(), "a write outside the pieces"
    assert torch.equal(_bits(p_local), _bits(p_before)), "the local parameters are not a destination"
    if not loose:
        for st, rs in zip(states, ref_states):
            for k in st:
                assert torch.equal(_bits(st[k]), _bits(rs[k])), k


def _lion_fp32_bounds(offs, g, p0, states0, got_p, want_p, got_s, want_s):
    """fp32 parameters, 32-bit Lion state (beta1, beta2 of _OPTS, lr 1e-3, weight decay 0.01): the parameter p0 (1 - lr
    wd) - lr sign(z), z = beta1 m + (1 - beta1) g, and the state beta2 m + (1 - beta2) g, each rounded once or twice
    depending on the contraction: within 2^-23 of the magnitudes that enter them.  Where z is within rounding of zero
    its sign may differ (one step, 2 lr, more); those elements must be rare."""
    b1, b2 = _OPTS["lion"]
    lr, eps = 1e-3, 2.0 ** -23
    near, total = 0, 0
    for i, (o, n) in enumerate(zip(offs, _PIECES)):
        gv, p, m = g[o:o + n].double(), p0[o:o + n].double(), states0[i].double()
        z_scale = (b1 * m).abs() + ((1 - b1) * gv).abs()
        flip = (b1 * m + (1 - b1) * gv).abs() <= 4 * eps * z_scale
        dp = (got_p[o:o + n].double() - want_p[o:o + n].double()).abs()
        bound = eps * (p.abs() + lr) + flip * 2 * lr
        ok = (dp <= bound) | (got_p[o:o + n].isnan() & want_p[o:o + n].isnan())
        assert ok.all(), ("parameters", i, dp[~ok][:4].tolist(), bound[~ok][:4].tolist())
        gs, ws = got_s[i]["state1"].double(), want_s[i]["state1"].double()
        finite = torch.isfinite(ws)
        assert torch.equal(finite, torch.isfinite(gs)) and torch.equal(gs.isnan(), ws.isnan()), ("state", i)
        ds = (gs - ws)[finite].abs()
        sbound = (eps * ((b2 * m).abs() + ((1 - b2) * gv).abs()))[finite]
        assert (ds <= sbound).all(), ("state", i, ds.max().item())
        near += int(flip.sum())
        total += n
    assert near <= total // 100, (near, total)


@pytest.mark.parametrize("w", range(1, 9))
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("eight", [True, False])
@pytest.mark.parametrize("name", list(_OPTS))
def test_peer_entry_equals_multi_on_reduced_gradient(name, eight, dtype, w):
    _check(name, dtype, eight, w, shift=0, scale=1.0 / 3.0)


@pytest.mark.parametrize("w", [1, 3, 8])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("eight", [True, False])
@pytest.mark.parametrize("name", ["adam", "lion"])
def test_misaligned_buffers_take_the_element_path(name, eight, dtype, w):
    _check(name, dtype, eight, w, shift=1, scale=1.0)


def test_rejected_arguments_write_nothing():
    """Bad counts and ids return 100, bad peers / bases / pieces 1, each with the message set; nothing is written."""
    td = torch.bfloat16
    offs, numel, grads, g_local, p_local, states = _case("adam", td, True, 2, 0, seed=1)
    dst = torch.full((numel,), float("nan"), dtype=td, device="cuda")
    d = cext.OptimTensor(p_local[offs[0]:].data_ptr(), g_local[offs[0]:].data_ptr(), states[0]["state1"].data_ptr(),
                         states[0]["state2"].data_ptr(), states[0]["absmax1"].data_ptr(),
                         states[0]["absmax2"].data_ptr(), _PIECES[0], 1, 0)
    q1, q2 = F.create_dynamic_map(signed=True).cuda(), F.create_dynamic_map(signed=False).cuda()
    s1_before = states[0]["state1"].clone()

    def call(opt=0, dtype=2, count=1, srcs=None, world=2, dsts=None, ndst=1, gl=None, pl=None, numel_=numel, q=True):
        srcs = [g.data_ptr() for g in grads] if srcs is None else srcs
        dsts = [dst.data_ptr()] if dsts is None else dsts
        a = (ct.c_void_p * max(1, len(srcs)))(*srcs)
        b = (ct.c_void_p * max(1, len(dsts)))(*dsts)
        rc = nat.lib.cbnb_b200_optimizer_update_8bit_blockwise_multi_peers(
            opt, dtype, ct.addressof(d), count, ct.cast(a, ct.c_void_p), world, ct.cast(b, ct.c_void_p), ndst,
            g_local.data_ptr() if gl is None else gl, p_local.data_ptr() if pl is None else pl, numel_, 0.5, 0.9,
            0.999, 0.0, 0.0, 1e-8, 0.0, 1e-3, q1.data_ptr() if q else None, q2.data_ptr() if q else None, False,
            torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return rc

    bad100 = [dict(count=-1), dict(count=10_000), dict(opt=6), dict(dtype=3)]
    bad1 = [dict(opt=5), dict(world=0), dict(world=9), dict(ndst=0), dict(ndst=9),
            dict(srcs=[grads[0].data_ptr(), 0]), dict(srcs=[grads[0].data_ptr() + 1, grads[1].data_ptr()]),
            dict(dsts=[0]), dict(dsts=[dst.data_ptr() + 1]), dict(gl=0), dict(pl=p_local.data_ptr() + 1),
            dict(numel_=offs[0] + _PIECES[0] - 1), dict(gl=g_local[offs[0] + 2:].data_ptr()), dict(q=False)]
    for kw in bad100:
        assert call(**kw) == 100, kw
        with pytest.raises(RuntimeError):
            nat.check()
    for kw in bad1:
        assert call(**kw) == 1, kw
        with pytest.raises(RuntimeError, match="peers"):
            nat.check()
    assert torch.isnan(dst).all() and torch.equal(states[0]["state1"], s1_before)
    assert call() == 0
    nat.check()
    assert not torch.isnan(dst[offs[0]:offs[0] + _PIECES[0]]).any()
    for kw in [dict(grad_srcs=[]), dict(grad_srcs=[grads[0].data_ptr()] * 9), dict(param_dsts=[0]),
               dict(grad_local=g_local[1:])]:
        args = dict(grad_srcs=[g.data_ptr() for g in grads], param_dsts=[dst.data_ptr()], grad_local=g_local)
        args.update(kw)
        with pytest.raises(ValueError):
            optimizer_update_8bit_blockwise_multi_peers(
                "adam", [g_local[offs[0]:offs[0] + _PIECES[0]]], [p_local[offs[0]:offs[0] + _PIECES[0]]],
                [states[0]["state1"]], [states[0]["state2"]], 0.9, 0.999, 0.0, 0.0, 1e-8, [1], 1e-3, q1, q2,
                [states[0]["absmax1"]], [states[0]["absmax2"]], 0.0, args["grad_srcs"], args["param_dsts"],
                args["grad_local"], p_local, 0.5)


# ------------------------------------------------------------------------------------------ processes
_SCRIPT = r"""
import copy, os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import bitsandbytes_b200 as bnb

rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
KEY = bnb.optim.optimizer.Optimizer8bit._FSDP_WRAPPED_QUANT_STATE_KEY


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


def same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b)), f"rank {rank}: {what}"


class Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(256, 384).to(torch.bfloat16)      # 8-bit weight, 32-bit bias
        self.b = torch.nn.Linear(384, 300).to(torch.bfloat16)      # weight spans both ranks
        self.n = torch.nn.LayerNorm(300)                           # fp32, 32-bit state
        self.c = torch.nn.Linear(300, 5000, bias=False)            # fp32, 8-bit
        self.frozen = torch.nn.Parameter(torch.ones(3), requires_grad=False)

    def forward(self, x):
        h = self.b(torch.relu(self.a(x.to(torch.bfloat16))))
        return self.c(self.n(h.float()))


def make(seed=0):
    torch.manual_seed(seed)
    return Net().to(dev)


MAKERS = {"AdamW8bit": lambda p: bnb.optim.AdamW8bit(p, lr=1e-3, weight_decay=0.01, min_8bit_size=4096),
          "Lion8bit": lambda p: bnb.optim.Lion8bit(p, lr=1e-4, min_8bit_size=4096),
          "SGD8bit": lambda p: bnb.optim.SGD8bit(p, lr=1e-2, momentum=0.9, min_8bit_size=4096),
          "RMSprop8bit": lambda p: bnb.optim.RMSprop8bit(p, lr=1e-4, min_8bit_size=4096),
          "Adagrad8bit": lambda p: bnb.optim.Adagrad8bit(p, lr=1e-3, min_8bit_size=4096),
          "Adam32bit": lambda p: bnb.optim.Adam32bit(p, lr=1e-3)}


def batch(step, micro):
    g = torch.Generator().manual_seed(1000 * step + 10 * micro + rank)
    return torch.randn(16, 256, generator=g).to(dev), torch.randn(16, 5000, generator=g).to(dev)


def reduced(t, scale):
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous())
    acc = parts[0].float()
    for q in parts[1:]:
        acc = acc + q.float()
    return (acc * torch.tensor(scale, dtype=torch.float32, device=dev)).to(t.dtype)


def train_step(model, opt, sched, ref, ref_opt, ref_sched, step, scale):
    for micro in range(2):                 # gradient accumulation over two micro-batches
        x, y = batch(step, micro)
        torch.nn.functional.mse_loss(model(x), y).backward()
    if step == 1:                          # a parameter without a gradient: updated with zeros
        model.n.bias.grad = None
    if ref is not None:
        for p, q in zip(model.parameters(), ref.parameters()):
            if p.requires_grad:
                q.grad = reduced(p.grad if p.grad is not None else torch.zeros_like(p), scale)
        ref_opt.step(); ref_opt.zero_grad(); ref_sched.step()
    opt.step(); opt.zero_grad(); sched.step()


def run(kind, steps=3, scale=None):
    model = make()
    ref = copy.deepcopy(model)
    if rank > 0:
        with torch.no_grad():
            for p in model.parameters():
                p.add_(1.0)                # rank 0's values win at construction
    opt = bnb.optim.ShardedOptimizer(MAKERS[kind](model.parameters()), grad_scale=scale)
    scale = opt.grad_scale
    ref_opt = MAKERS[kind](ref.parameters())
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=0.5)
    ref_sched = torch.optim.lr_scheduler.StepLR(ref_opt, step_size=1, gamma=0.5)
    for step in range(steps):
        train_step(model, opt, sched, ref, ref_opt, ref_sched, step, scale)
        for (name, p), q in zip(model.named_parameters(), ref.parameters()):
            same(p.detach(), q.detach(), f"{kind} step {step} {name}")
    for f in opt.flats:                    # identical on every rank
        every = [torch.empty_like(f.param) for _ in range(world)]
        dist.all_gather(every, f.param)
        for e in every:
            same(e, f.param, f"{kind}: ranks differ")
    full = opt.consolidated_state_dict()
    assert (full is None) == (rank != 0)
    box = [full]
    dist.broadcast_object_list(box, src=0)
    full = box[0]
    want = ref_opt.state_dict()
    assert set(full["state"]) == set(want["state"]), (sorted(full["state"]), sorted(want["state"]))
    for k, v in want["state"].items():
        assert full["state"][k]["step"] == v["step"], (k, full["state"][k]["step"], v["step"])
        got = full["state"][k][KEY]
        assert set(got) == set(v[KEY]), (set(got), set(v[KEY]))
        for key, t in v[KEY].items():
            assert got[key].device.type == "cpu"
            same(got[key].to(dev), t, f"{kind} consolidated {k} {key}")
    return model, opt, ref, ref_opt, full


def checkpoint(kind):
    # the consolidated state loads into a plain optimizer and back into a sharded one; both train on with equal bits
    model, opt, ref, ref_opt, full = run(kind)
    plain_model = copy.deepcopy(ref)
    plain = MAKERS[kind](plain_model.parameters())
    plain.load_state_dict(full)
    model2 = copy.deepcopy(ref)
    opt2 = bnb.optim.ShardedOptimizer(MAKERS[kind](model2.parameters()))
    opt2.load_state_dict(full)
    shard = opt2.state_dict()
    opt2.load_state_dict(shard)
    s1 = torch.optim.lr_scheduler.StepLR(plain, step_size=1, gamma=1.0)
    s2 = torch.optim.lr_scheduler.StepLR(opt2, step_size=1, gamma=1.0)
    for step in range(3, 5):
        train_step(model2, opt2, s2, plain_model, plain, s1, step, opt2.grad_scale)
        for p, q in zip(model2.parameters(), plain_model.parameters()):
            same(p.detach(), q.detach(), f"{kind} reloaded step {step}")


for kind in MAKERS:
    run(kind, scale=1.0 if kind == "SGD8bit" else None)
for kind in ("AdamW8bit", "Lion8bit", "Adam32bit"):
    checkpoint(kind)
dist.barrier()
dist.destroy_process_group()
print("SHARDED_OK", rank)
"""


@pytest.mark.parametrize("nproc", [1, 2])
def test_processes_sharded_training_equals_unsharded(tmp_path, nproc):
    """One process per GPU: every supported class (8-bit and 32-bit, bf16 and fp32 tensors) trains three steps with
    gradient accumulation and a StepLR; parameters equal the unsharded optimizer's fed the rank-order-reduced gradient
    after every step, on every rank; the consolidated state equals the unsharded optimizer's state dict; it reloads
    into a plain and a sharded optimizer that train on equally."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "sharded.py"
    script.write_text(_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29671 + nproc), str(script)],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and r.stdout.count("SHARDED_OK") == nproc, r.stdout[-3000:] + r.stderr[-4000:]
