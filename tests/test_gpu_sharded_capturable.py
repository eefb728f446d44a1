"""GPU tests of the capturable data-parallel step (``ShardedOptimizer`` over an optimizer made with ``capturable=True``;
the ``_peers_dev`` entries of csrc/c_api.cu).

* The entries, with w "ranks" simulated as separate buffers passed as raw addresses (as test_gpu_sharded_optim.py):
  with device counters holding k and ``lr_dev`` = lr, the bits of the host-step entries with step k and that lr, for
  every optimizer, dtype, state width, w in {1, 2, 5, 8}, with and without the clip coefficient; misaligned buffers;
  the counters are read and not advanced; a NULL counter is refused.
* In one process: a capturable ShardedOptimizer stepped eagerly equals a non-capturable one, bit for bit; one captured
  ``step()`` replayed k times (new gradients copied in between) equals k eager steps, also with a tensor lr that a
  scheduler changes between replays and with ``clip_grad_norm_`` inside the captured region.
* One process per GPU (torch.distributed.run, 1 and 2 processes): a whole data-parallel QLoRA iteration (forward
  through Linear4bit plus LoRA adapters, backward, clip, step, zero_grad, NCCL collectives included) captured in one
  graph and replayed equals the same iterations run eagerly, and the unsharded optimizer fed the mean gradient.
"""
import ctypes as ct
import os
import subprocess
import sys

import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.functional as F
from bitsandbytes_b200.backends import cuda as backend
from bitsandbytes_b200.backends.cuda import (optimizer_update_32bit_multi_peers,
                                             optimizer_update_8bit_blockwise_multi_peers)
from tests import _native as nat
from tests.test_gpu_sharded_optim import _DT, _OPTS, _PIECES, _bits, _case

pytestmark = pytest.mark.gpu

_QK = "__bnb_optimizer_quant_state__"
_LR = float(torch.tensor(1e-3, dtype=torch.float32))  # an fp32 value: lr_dev holds the same number


def _update(name, eight, offs, g_local, p_local, states, srcs, dsts, scale, steps, lr, coef):
    b1, b2 = _OPTS[name]
    g = [g_local[o:o + n] for o, n in zip(offs, _PIECES)]
    p = [p_local[o:o + n] for o, n in zip(offs, _PIECES)]
    s1 = [st["state1"] for st in states]
    s2 = [st["state2"] for st in states] if name == "adam" else None
    kw = {} if coef is None else {"gnorm_scale_dev": coef}
    if eight:
        q1, q2 = F.create_dynamic_map(signed=True).cuda(), F.create_dynamic_map(signed=False).cuda()
        optimizer_update_8bit_blockwise_multi_peers(name, g, p, s1, s2, b1, b2, 0.0, 0.0, 1e-8, steps, lr, q1, q2,
                                                    [st["absmax1"] for st in states],
                                                    [st["absmax2"] for st in states] if s2 else None, 0.01, srcs,
                                                    dsts, g_local, p_local, scale, **kw)
    else:
        optimizer_update_32bit_multi_peers(name, g, p, s1, s2, b1, b2, 0.0, 0.0, 1e-8, 0.01, steps, lr, srcs, dsts,
                                           g_local, p_local, scale, **kw)


def _entry_check(name, dtype, eight, w, shift, coef, lr_tensor=True):
    td = _DT[dtype]
    offs, numel, grads, g_local, p_local, states = _case(name, td, eight, w, shift, seed=w * 13 + shift + 2)
    ref_states = [{k: v.clone() for k, v in st.items()} for st in states]
    p_before = p_local.clone()
    c = None if coef is None else torch.full((1,), coef, dtype=torch.float32, device="cuda")
    host_steps = [3 + 5 * i for i in range(len(_PIECES))]
    counters = torch.tensor(host_steps, dtype=torch.int32, device="cuda")
    lr = torch.full((1,), _LR, dtype=torch.float32, device="cuda") if lr_tensor else _LR

    def dests():
        return [torch.full((numel + shift,), float("nan"), dtype=td, device="cuda")[shift:] for _ in range(w)]

    srcs = [t.data_ptr() for t in grads]
    want, got = dests(), dests()
    _update(name, eight, offs, g_local, p_local, ref_states, srcs, [d.data_ptr() for d in want], 1.0 / 3.0,
            host_steps, _LR, c)
    _update(name, eight, offs, g_local, p_local, states, srcs, [d.data_ptr() for d in got], 1.0 / 3.0,
            list(counters.split(1)), lr, c)
    torch.cuda.synchronize()
    assert counters.tolist() == host_steps, "the _peers_dev entries read the counters and do not advance them"
    for a, b in zip(got, want):
        assert torch.equal(_bits(a), _bits(b)), "parameters"
    assert torch.equal(_bits(p_local), _bits(p_before))
    for st, rs in zip(states, ref_states):
        for k in st:
            assert torch.equal(_bits(st[k]), _bits(rs[k])), k


@pytest.mark.parametrize("coef", [None, 0.37])
@pytest.mark.parametrize("w", [1, 2, 5, 8])
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("eight", [True, False])
@pytest.mark.parametrize("name", list(_OPTS))
def test_dev_entries_equal_host_step_entries(name, eight, dtype, w, coef):
    _entry_check(name, dtype, eight, w, shift=0, coef=coef)


@pytest.mark.parametrize("w", [1, 3])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("eight", [True, False])
@pytest.mark.parametrize("name", ["adam", "lion"])
def test_dev_entries_misaligned_and_lr_by_value(name, eight, dtype, w):
    _entry_check(name, dtype, eight, w, shift=1, coef=0.5)
    _entry_check(name, dtype, eight, w, shift=0, coef=None, lr_tensor=False)


def test_null_counter_is_refused_and_nothing_written():
    td = torch.bfloat16
    offs, numel, grads, g_local, p_local, states = _case("adam", td, True, 2, 0, seed=4)
    counters = torch.ones(len(_PIECES), dtype=torch.int32, device="cuda")
    g = [g_local[o:o + n] for o, n in zip(offs, _PIECES)]
    p = [p_local[o:o + n] for o, n in zip(offs, _PIECES)]
    _, descs, dev = backend._optimizer_list("t", "adam", backend._OPTIMIZER_ID, g, p, [s["state1"] for s in states],
                                            [s["state2"] for s in states], [s["absmax1"] for s in states],
                                            [s["absmax2"] for s in states], list(counters.split(1)), True)
    assert dev
    descs[2].step_ptr = None
    dst = torch.full((numel,), float("nan"), dtype=td, device="cuda")
    s1 = states[0]["state1"].clone()
    q1, q2 = F.create_dynamic_map(signed=True).cuda(), F.create_dynamic_map(signed=False).cuda()
    srcs = (ct.c_void_p * 2)(*[t.data_ptr() for t in grads])
    dsts = (ct.c_void_p * 1)(dst.data_ptr())
    stream = torch.cuda.current_stream().cuda_stream
    rc = nat.lib.cbnb_b200_optimizer_update_8bit_blockwise_multi_peers_dev(
        0, 2, ct.addressof(descs), len(_PIECES), ct.cast(srcs, ct.c_void_p), 2, ct.cast(dsts, ct.c_void_p), 1,
        g_local.data_ptr(), p_local.data_ptr(), numel, 0.5, 0.9, 0.999, 0.0, 0.0, 1e-8, 0.0, 1e-3, q1.data_ptr(),
        q2.data_ptr(), False, None, None, stream)
    assert rc == 100
    with pytest.raises(RuntimeError, match="step_ptr"):
        nat.check()
    rc = nat.lib.cbnb_b200_optimizer_update_32bit_multi_peers_dev(
        0, 2, ct.addressof(descs), len(_PIECES), ct.cast(srcs, ct.c_void_p), 2, ct.cast(dsts, ct.c_void_p), 1,
        g_local.data_ptr(), p_local.data_ptr(), numel, 0.5, 0.9, 0.999, 0.0, 0.0, 1e-8, 0.0, 1e-3, False, None, None,
        stream)
    assert rc == 100
    with pytest.raises(RuntimeError, match="step_ptr"):
        nat.check()
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.equal(states[0]["state1"], s1)
    assert counters.tolist() == [1] * len(_PIECES)


# ------------------------------------------------------------------------------------------ one process
# bf16 and fp32 tensors, 8-bit (from 4096 elements) and 32-bit state, a ragged last block and an empty tensor
_SHAPES = [((96, 64), torch.bfloat16), ((300,), torch.bfloat16), ((0,), torch.bfloat16), ((5000,), torch.float32),
           ((7,), torch.float32), ((33, 129), torch.bfloat16)]
_MAKERS = {"AdamW8bit": lambda p, lr, c: bnb.optim.AdamW8bit(p, lr=lr, weight_decay=0.01, capturable=c),
           "Lion8bit": lambda p, lr, c: bnb.optim.Lion8bit(p, lr=lr, capturable=c),
           "SGD8bit": lambda p, lr, c: bnb.optim.SGD8bit(p, lr=lr, momentum=0.9, capturable=c),
           "AdamW": lambda p, lr, c: bnb.optim.AdamW(p, lr=lr, capturable=c),
           "RMSprop": lambda p, lr, c: bnb.optim.RMSprop(p, lr=lr, capturable=c)}


def _params():
    gen = torch.Generator().manual_seed(0)
    return [torch.nn.Parameter((torch.randn(*s, generator=gen) * 0.5).to(dt).cuda()) for s, dt in _SHAPES]


def _grads(k):
    gen = torch.Generator().manual_seed(100 + k)
    scale = 4.0 if k % 2 else 0.25  # some steps clip at max_norm 1, some do not
    return [(torch.randn(*s, generator=gen) * scale).to(dt).cuda() for s, dt in _SHAPES]


def _lrs(k):
    return float(torch.tensor(1e-3 * (1.0 - 0.1 * k), dtype=torch.float32))


def _equal(a, b):
    pa, pb = [p for g in a.param_groups for p in g["params"]], [p for g in b.param_groups for p in g["params"]]
    for x, y in zip(pa, pb):
        assert torch.equal(_bits(x.detach()), _bits(y.detach()))
    sa, sb = a.consolidated_state_dict(), b.consolidated_state_dict()
    for k in sa["state"]:
        assert sa["state"][k]["step"] == sb["state"][k]["step"]
        wa, wb = sa["state"][k][_QK], sb["state"][k][_QK]
        for key in wa:
            assert torch.equal(_bits(wa[key]), _bits(wb[key])), (k, key)


def _eager(kind, k_steps, clip, capturable, tensor_lr, vary_lr=True):
    """A sharded optimizer after k eager steps (gradients _grads(k), lr _lrs(k) or, without vary_lr, _lrs(0))."""
    lr = torch.full((1,), _lrs(0), device="cuda") if tensor_lr else _lrs(0)
    opt = bnb.optim.ShardedOptimizer(_MAKERS[kind](_params(), lr, capturable))
    for k in range(k_steps):
        if vary_lr:
            _set_lr(opt, k)
        for p, g in zip(opt.param_groups[0]["params"], _grads(k)):
            p.grad.copy_(g)
        if clip:
            opt.clip_grad_norm_(1.0)
        opt.step()
    return opt


def _set_lr(opt, k):
    g = opt.param_groups[0]
    if isinstance(g["lr"], torch.Tensor):
        g["lr"].fill_(_lrs(k))   # a scheduler writing the tensor in place
    else:
        g["lr"] = _lrs(k)


@pytest.mark.parametrize("kind", list(_MAKERS))
def test_capturable_eager_equals_non_capturable(kind):
    plain = _eager(kind, 4, clip=True, capturable=False, tensor_lr=False)
    cap = _eager(kind, 4, clip=True, capturable=True, tensor_lr=True)
    assert cap.steps.tolist() == [4] * len(_SHAPES)
    _equal(cap, plain)


@pytest.mark.parametrize("mode", ["float_lr", "tensor_lr", "clip"])
@pytest.mark.parametrize("kind", list(_MAKERS))
def test_captured_step_replays_equal_eager_steps(kind, mode):
    k_steps = 6
    clip, tensor_lr = mode == "clip", mode != "float_lr"
    ref = _eager(kind, k_steps, clip, capturable=False, tensor_lr=False, vary_lr=tensor_lr)
    lr = torch.full((1,), _lrs(0), device="cuda") if tensor_lr else _lrs(0)
    opt = bnb.optim.ShardedOptimizer(_MAKERS[kind](_params(), lr, True))
    params = opt.param_groups[0]["params"]

    def region():
        if clip:
            opt.clip_grad_norm_(1.0)
        opt.step()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # step 0, eager: makes the clip's buffers
        for p, g in zip(params, _grads(0)):
            p.grad.copy_(g)
        region()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        region()
    for k in range(1, k_steps):
        if tensor_lr:
            _set_lr(opt, k)
        for p, g in zip(params, _grads(k)):
            p.grad.copy_(g)
        graph.replay()
    torch.cuda.synchronize()
    assert opt.steps.tolist() == [k_steps] * len(_SHAPES)
    _equal(opt, ref)  # (a float lr was captured: the reference keeps it too)


def test_capture_refusals_and_a_load_under_a_captured_graph():
    opt = bnb.optim.ShardedOptimizer(_MAKERS["AdamW8bit"](_params(), _lrs(0), True))
    with pytest.raises(RuntimeError, match="run one eager"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            opt.clip_grad_norm_(1.0)
    plain = bnb.optim.ShardedOptimizer(_MAKERS["AdamW8bit"](_params(), _lrs(0), False))
    with pytest.raises(RuntimeError, match="capturable=False"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            plain.step()
    opt.step()
    sd = opt.state_dict()                 # after one step (the live state tensors: cloned)
    sd["pieces"] = [dict(q, state={k: v.clone() for k, v in q["state"].items()}) for q in sd["pieces"]]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    assert opt.steps.tolist() == [3] * len(_SHAPES)
    opt.load_state_dict(sd)               # in place: the graph continues from the loaded step
    graph.replay()
    torch.cuda.synchronize()
    assert opt.steps.tolist() == [2] * len(_SHAPES)
    again = bnb.optim.ShardedOptimizer(_MAKERS["AdamW8bit"](_params(), _lrs(0), False))
    again.step()
    again.step()
    st_a, st_b = opt.state_dict(), again.state_dict()
    assert st_a["steps"] == st_b["steps"]
    for qa, qb in zip(st_a["pieces"], st_b["pieces"]):
        for key in qa["state"]:
            assert torch.equal(_bits(qa["state"][key]), _bits(qb["state"][key])), key


# ------------------------------------------------------------------------------------------ processes
_SCRIPT = r"""
import math, os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import bitsandbytes_b200 as bnb
import bitsandbytes_b200.optim.optimizer as bopt

rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
F = bopt.F
QK = "__bnb_optimizer_quant_state__"


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


class Scaled:
    # the unsharded optimizer's launches with gnorm_scale set to the clip coefficient
    def __init__(self, coef):
        self.coef = coef

    def __getattr__(self, name):
        return getattr(F, name)

    def optimizer_update_32bit_multi(self, *a, **kw):
        a = list(a)
        a[13] = self.coef
        return F.optimizer_update_32bit_multi(*a, **kw)

    def optimizer_update_8bit_blockwise_multi(self, *a, **kw):
        kw["gnorm_scale"] = self.coef
        return F.optimizer_update_8bit_blockwise_multi(*a, **kw)


class LoRALinear4bit(torch.nn.Module):
    def __init__(self, k, n, r, gen):
        super().__init__()
        lin = torch.nn.Linear(k, n, bias=False)
        with torch.no_grad():
            lin.weight.copy_(torch.randn(n, k, generator=gen) / k**0.5)
        self.base = bnb.nn.Linear4bit(k, n, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4")
        self.base.load_state_dict(lin.state_dict())
        self.base = self.base.to(dev)
        self.A = torch.nn.Parameter((torch.randn(r, k, generator=gen) / k**0.5).to(torch.bfloat16).to(dev))
        self.B = torch.nn.Parameter((torch.randn(n, r, generator=gen) * 0.01).to(torch.bfloat16).to(dev))

    def forward(self, x):
        return self.base(x) + (x @ self.A.t()) @ self.B.t()


def model():
    gen = torch.Generator().manual_seed(9)
    return torch.nn.Sequential(LoRALinear4bit(1024, 1024, 16, gen), LoRALinear4bit(1024, 512, 16, gen))


def reduced(t, scale):
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous())
    acc = parts[0].float()
    for q in parts[1:]:
        acc = acc + q.float()
    return (acc * torch.tensor(scale, dtype=torch.float32, device=dev)).to(t.dtype)


def trainable(m):
    return [p for p in m.parameters() if p.requires_grad]


MAKERS = {"AdamW8bit": lambda p, c: bnb.optim.AdamW8bit(p, lr=1e-3, weight_decay=0.01, capturable=c),
          "AdamW": lambda p, c: bnb.optim.AdamW(p, lr=1e-3, capturable=c)}
M, K, MAX_NORM = 64, 7, 0.05
for kind, make in MAKERS.items():
    gen = torch.Generator().manual_seed(1000 + rank)
    data = [(torch.randn(M, 1024, generator=gen).to(torch.bfloat16).to(dev),
             torch.randn(M, 512, generator=gen).to(torch.bfloat16).to(dev)) for _ in range(K)]
    ma, mb, mc = model(), model(), model()
    for m in (ma, mb, mc):
        for p in m.parameters():
            if p.dtype == torch.uint8:
                p.requires_grad_(False)
    oa = bnb.optim.ShardedOptimizer(make(trainable(ma), True))
    ob = bnb.optim.ShardedOptimizer(make(trainable(mb), False))
    oc = make(trainable(mc), False)

    def iteration(m, opt, x, y):
        loss = torch.nn.functional.mse_loss(m(x), y)
        loss.backward()
        total = opt.clip_grad_norm_(MAX_NORM)
        opt.step()
        opt.zero_grad()
        return loss, total

    # the eager runs: ob (sharded, not capturable) and oc (unsharded, fed the mean gradient and the coefficient)
    clipped = 0
    for x, y in data:
        loss = torch.nn.functional.mse_loss(mb(x), y)
        loss.backward()
        reds = [reduced(p.grad, ob.grad_scale) for p in trainable(mb)]
        total = ob.clip_grad_norm_(MAX_NORM)
        ob.step()
        ob.zero_grad()
        coef = float((MAX_NORM / (total.reshape(1).clone() + 1e-6)).clamp(max=1.0))
        clipped += coef < 1.0
        torch.nn.functional.mse_loss(mc(x), y).backward()
        for q, r in zip(trainable(mc), reds):
            q.grad = r
        bopt.F = Scaled(coef)
        try:
            oc.step()
        finally:
            bopt.F = F
        oc.zero_grad()
    assert clipped, "no iteration clipped"
    # the captured run: one eager iteration, then one graph replayed on fresh static inputs
    static_x, static_y = data[0][0].clone(), data[0][1].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        iteration(ma, oa, static_x, static_y)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss, static_total = iteration(ma, oa, static_x, static_y)
    for x, y in data[1:]:
        static_x.copy_(x)
        static_y.copy_(y)
        graph.replay()
    torch.cuda.synchronize()
    assert oa.steps.tolist() == [K] * len(oa.entries)
    for (name, a), b, c in zip(ma.named_parameters(), mb.parameters(), mc.parameters()):
        assert torch.equal(bits(a.detach()), bits(b.detach())), f"rank {rank} {kind} {name}: graph != eager"
        if a.requires_grad:
            assert torch.equal(bits(b.detach()), bits(c.detach())), f"rank {rank} {kind} {name}: sharded != unsharded"
    sa, sb = oa.consolidated_state_dict(), ob.consolidated_state_dict()
    if rank == 0:
        sc = oc.state_dict()
        for k in sa["state"]:
            assert sa["state"][k]["step"] == sb["state"][k]["step"] == sc["state"][k]["step"] == K
            for key, v in sa["state"][k][QK].items():
                assert torch.equal(bits(v), bits(sb["state"][k][QK][key])), (kind, k, key, "graph != eager")
                assert torch.equal(bits(v), bits(sc["state"][k][QK][key].cpu())), (kind, k, key, "!= unsharded")
    del graph
dist.barrier()
dist.destroy_process_group()
print("GRAPH_OK", rank)
"""


@pytest.mark.parametrize("nproc", [1, 2])
def test_processes_captured_qlora_iteration_equals_eager(tmp_path, nproc):
    """One process per GPU: AdamW8bit and AdamW (32-bit) over the LoRA adapters of two 4-bit layers; an iteration
    (forward, backward, clip_grad_norm_, step, zero_grad) captured in one CUDA graph with its all-to-all and
    all-gathers, replayed on new inputs, equals bit for bit the eager sharded iterations (parameters and consolidated
    state) and the unsharded optimizer fed the mean gradient with gnorm_scale = the clip coefficient."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "graph.py"
    script.write_text(_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29731 + nproc), str(script)],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and r.stdout.count("GRAPH_OK") == nproc, r.stdout[-3000:] + r.stderr[-4000:]
