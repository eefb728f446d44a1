"""GPU tests of capturable optimizer steps (``capturable=True``: device step counters, an optional device learning
rate, the _dev kernels of csrc/optim.cu):

* eager capturable steps equal ``capturable=False`` steps bit for bit, for every class of test_gpu_optim_multi.py that
  can be capturable, on a mixed list (fp32 / fp16 / bf16 parameters, a ragged last 256-block, 32-bit state below
  min_8bit_size);
* the replays of one captured ``step()`` equal eager steps on the same gradients, bit for bit, and advance the steps;
* a tensor lr driven by ``LambdaLR`` between replays; a list longer than one launch; a state_dict round trip through a
  plain optimizer; the capture guard;
* a whole QLoRA step (NF4 ``Linear4bit`` base, LoRA A / B, forward, backward and ``AdamW8bit``) captured as one graph.
"""
import pytest
import torch

import bitsandbytes_b200 as bnb
from bitsandbytes_b200.backends.cuda import optimizer_multi_capacity

pytestmark = pytest.mark.gpu

# the classes of test_gpu_optim_multi.py, without paged state and AdEMAMix's schedules (refused when capturable)
CLASSES = {
    "Adam8bit": (bnb.optim.Adam8bit, dict(lr=1e-3)),
    "AdamW8bit": (bnb.optim.AdamW8bit, dict(lr=1e-3)),
    "Lion8bit": (bnb.optim.Lion8bit, dict(lr=1e-4)),
    "AdEMAMix8bit": (bnb.optim.AdEMAMix8bit, dict(lr=1e-3)),
    "RMSprop8bit": (bnb.optim.RMSprop8bit, dict(lr=1e-3)),
    "Adagrad8bit": (bnb.optim.Adagrad8bit, dict(lr=1e-2)),
    "SGD8bit": (bnb.optim.SGD8bit, dict(lr=1e-2, momentum=0.9)),
    "Adam": (bnb.optim.Adam, dict(lr=1e-3)),
    "AdamW": (bnb.optim.AdamW, dict(lr=1e-3)),
    "Lion": (bnb.optim.Lion, dict(lr=1e-4)),
    "AdEMAMix": (bnb.optim.AdEMAMix, dict(lr=1e-3)),
    "RMSprop": (bnb.optim.RMSprop, dict(lr=1e-3)),
    "Adagrad": (bnb.optim.Adagrad, dict(lr=1e-2)),
    "SGD": (bnb.optim.SGD, dict(lr=1e-2, momentum=0.9)),
}
# 8-bit state from 4096 elements (min_8bit_size); (33, 129) and (5000,) end in a ragged 256-block (left out for
# AdEMAMix8bit, whose slow EMA needs n % 256 == 0 above min_8bit_size: see test_gpu_optim_multi.py)
SHAPES = [((64, 64), torch.float32), ((4095,), torch.float32), ((33, 129), torch.bfloat16), ((300,), torch.float16),
          ((80, 64), torch.float16), ((96, 256), torch.bfloat16), ((65,), torch.bfloat16), ((5000,), torch.float16),
          ((7,), torch.float32), ((16, 256), torch.float32)]


def _params(name, seed=1):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    shapes = [(s, d) for s, d in SHAPES if not (name == "AdEMAMix8bit" and s in ((33, 129), (5000,)))]
    return [torch.nn.Parameter((torch.randn(s, generator=gen) * 0.1).to(d).cuda()) for s, d in shapes]


def _make(cls, params, kw, **extra):
    """Two parameter groups with different lr and weight decay."""
    half = len(params) // 2
    kw2 = dict(kw, lr=kw["lr"] * 2, weight_decay=0.05)
    return cls([{"params": params[:half]}, {"params": params[half:], **kw2}], **kw, **extra)


def _grads(params, gen):
    return [(torch.randn(p.shape, generator=gen) * 0.01).to(p.dtype).cuda() for p in params]


def _assert_same(oa, pa, ob, pb, what, step=None):
    for i, (x, y) in enumerate(zip(pa, pb)):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"{what}: parameter {i} differs"
        sa, sb = oa.state[x], ob.state[y]
        for k in ("state1", "state2", "absmax1", "absmax2"):
            assert (k in sa) == (k in sb), f"{what}: {k} of {i}"
            if k in sa:
                assert torch.equal(sa[k].view(torch.uint8), sb[k].view(torch.uint8)), f"{what}: {k} of parameter {i}"
        if step is not None:
            sc = sa["step"] if isinstance(sa["step"], torch.Tensor) else sb["step"]
            assert sc.dtype == torch.int32 and sc.is_cuda and int(sc.item()) == step, f"{what}: step of {i}"


@pytest.mark.parametrize("name", list(CLASSES))
def test_eager_capturable_steps_equal_plain_steps(name):
    cls, kw = CLASSES[name]
    pa, pb = _params(name), _params(name)
    oa, ob = _make(cls, pa, kw, capturable=True), _make(cls, pb, kw)
    gen = torch.Generator(device="cpu").manual_seed(2)
    for step in range(1, 5):
        for x, y, g in zip(pa, pb, _grads(pa, gen)):
            x.grad, y.grad = g.clone(), g.clone()
        oa.step()
        ob.step()
        torch.cuda.synchronize()
        _assert_same(oa, pa, ob, pb, f"{name} step {step}", step=step)
    kinds = [oa.state[p]["state1"].dtype for p in pa[:2]]  # 4096 / 4095 elements: either side of min_8bit_size
    assert kinds == ([torch.uint8, torch.float32] if name.endswith("8bit") else [torch.float32] * 2)


def _warm_up_and_capture(opt, params, twin, twin_params, gen, steps=2, between=None):
    """`steps` eager steps of both on a side stream (the capturable one through static .grad tensors), then capture one
    step() of `opt`.  Returns the graph."""
    for p in params:
        p.grad = torch.zeros_like(p)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(steps):
            for x, y, g in zip(params, twin_params, _grads(params, gen)):
                x.grad.copy_(g)
                y.grad = g.clone()
            opt.step()
            twin.step()
            if between is not None:
                between()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    return graph


def _replay(graph, params, twin, twin_params, gen, replays=5, between=None):
    for _ in range(replays):
        for x, y, g in zip(params, twin_params, _grads(params, gen)):
            x.grad.copy_(g)
            y.grad = g.clone()
        graph.replay()
        twin.step()
        if between is not None:
            between()
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", list(CLASSES))
def test_replays_of_a_captured_step_equal_eager_steps(name):
    cls, kw = CLASSES[name]
    pa, pb = _params(name), _params(name)
    oa, ob = _make(cls, pa, kw, capturable=True), _make(cls, pb, kw)
    gen = torch.Generator(device="cpu").manual_seed(3)
    graph = _warm_up_and_capture(oa, pa, ob, pb, gen)
    torch.cuda.synchronize()
    _assert_same(oa, pa, ob, pb, f"{name} after capture", step=2)  # (capturing launches nothing)
    _replay(graph, pa, ob, pb, gen)
    _assert_same(oa, pa, ob, pb, f"{name} after 5 replays", step=7)


@pytest.mark.parametrize("name", ["AdamW8bit", "AdamW", "Lion8bit", "SGD"])
def test_a_tensor_lr_follows_its_scheduler_between_replays(name):
    cls, kw = CLASSES[name]
    pa, pb = _params(name), _params(name)
    lr = torch.tensor(kw["lr"], dtype=torch.float32, device="cuda")
    oa = cls(pa, **dict(kw, lr=lr), capturable=True)
    ob = cls(pb, **kw)
    # powers of two: the float schedule rounded to fp32 and the fp32 tensor schedule are the same numbers
    sa = torch.optim.lr_scheduler.LambdaLR(oa, lambda e: 0.5 ** (e % 4))
    sb = torch.optim.lr_scheduler.LambdaLR(ob, lambda e: 0.5 ** (e % 4))

    def sched():
        sa.step()
        sb.step()

    gen = torch.Generator(device="cpu").manual_seed(4)
    graph = _warm_up_and_capture(oa, pa, ob, pb, gen, between=sched)
    _replay(graph, pa, ob, pb, gen, between=sched)
    assert oa.param_groups[0]["lr"] is lr and lr.item() == pytest.approx(ob.param_groups[0]["lr"], rel=1e-6)
    assert ob.param_groups[0]["lr"] != kw["lr"]
    _assert_same(oa, pa, ob, pb, f"{name} with a scheduled tensor lr", step=7)


@pytest.mark.parametrize("name", ["AdamW8bit", "AdamW"])
def test_a_captured_list_longer_than_one_launch(name):
    """1000 tensors of 1 .. 4800 elements: several launches, each with its own increment kernel."""
    cls, kw = CLASSES[name]
    cap = optimizer_multi_capacity()
    gen = torch.Generator(device="cpu").manual_seed(5)
    sizes = torch.randint(1, 4800, (1000,), generator=gen).tolist()
    assert len(sizes) > 2 * cap

    def params():
        g = torch.Generator(device="cpu").manual_seed(6)
        return [torch.nn.Parameter((torch.randn(n, generator=g) * 0.1).to(torch.bfloat16).cuda()) for n in sizes]

    pa, pb = params(), params()
    oa, ob = cls(pa, **kw, min_8bit_size=0, capturable=True), cls(pb, **kw, min_8bit_size=0)
    graph = _warm_up_and_capture(oa, pa, ob, pb, gen)
    _replay(graph, pa, ob, pb, gen)
    assert all(oa.state[p]["state1"].dtype == (torch.uint8 if name.endswith("8bit") else torch.float32) for p in pa)
    _assert_same(oa, pa, ob, pb, f"{name}, 1000 tensors", step=7)


@pytest.mark.parametrize("name", ["AdamW8bit", "Lion", "AdEMAMix8bit"])
def test_a_state_dict_round_trip_through_a_plain_optimizer(name):
    cls, kw = CLASSES[name]
    pa, pb = _params(name), _params(name)
    oa, ob = _make(cls, pa, kw, capturable=True), _make(cls, pb, kw, capturable=True)
    gen = torch.Generator(device="cpu").manual_seed(7)
    for step in range(1, 7):
        for x, y, g in zip(pa, pb, _grads(pa, gen)):
            x.grad, y.grad = g.clone(), g.clone()
        oa.step()
        ob.step()
        if step == 2:  # capturable -> plain
            sd = oa.state_dict()
            assert all(type(s["step"]) is int and s["step"] == 2 for s in sd["state"].values())
            oa = _make(cls, pa, kw)
            oa.load_state_dict(sd)
        elif step == 4:  # plain -> capturable
            sd = oa.state_dict()
            assert all(type(s["step"]) is int and s["step"] == 4 for s in sd["state"].values())
            oa = _make(cls, pa, kw, capturable=True)
            oa.load_state_dict(sd)
            assert all(oa.state[p]["step"].dtype == torch.int32 and oa.state[p]["step"].is_cuda for p in pa)
    torch.cuda.synchronize()
    _assert_same(ob, pb, oa, pa, f"{name} after the round trip", step=6)


def test_capturing_a_non_capturable_step_raises_before_any_launch():
    pa = _params("AdamW8bit")
    opt = bnb.optim.AdamW8bit(pa, lr=1e-3)
    for p in pa:
        p.grad = torch.randn_like(p) * 0.01
    opt.step()
    torch.cuda.synchronize()
    before = [p.detach().clone() for p in pa]
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="capturable=False"):
        with torch.cuda.graph(graph):
            opt.step()
    torch.cuda.synchronize()
    assert all(opt.state[p]["step"] == 1 for p in pa)
    assert all(torch.equal(p, b) for p, b in zip(pa, before))
    fresh = bnb.optim.AdamW8bit(pa, lr=1e-3, capturable=True)  # a capturable optimizer without state
    with pytest.raises(RuntimeError, match="run one eager step"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            fresh.step()
    assert all(len(fresh.state[p]) == 0 for p in pa)


# ------------------------------------------------------------------------------------------ a whole QLoRA step
class _LoRALinear4bit(torch.nn.Module):
    """A frozen NF4 Linear4bit (bf16 compute) plus trainable LoRA A / B."""

    def __init__(self, k, n, r, gen):
        super().__init__()
        lin = torch.nn.Linear(k, n, bias=False)
        with torch.no_grad():
            lin.weight.copy_(torch.randn(n, k, generator=gen) / k**0.5)
        self.base = bnb.nn.Linear4bit(k, n, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4")
        self.base.load_state_dict(lin.state_dict())
        self.base = self.base.cuda()
        self.A = torch.nn.Parameter((torch.randn(r, k, generator=gen) / k**0.5).to(torch.bfloat16).cuda())
        self.B = torch.nn.Parameter((torch.randn(n, r, generator=gen) * 0.01).to(torch.bfloat16).cuda())

    def forward(self, x):
        return self.base(x) + (x @ self.A.t()) @ self.B.t()


def _qlora(seed):
    """Two layers: the first layer's adapters get their gradient through the second layer's 4-bit base."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    return torch.nn.Sequential(_LoRALinear4bit(1024, 1024, 16, gen), _LoRALinear4bit(1024, 512, 16, gen))


def test_a_whole_qlora_step_captured_as_one_graph():
    M = 64
    ma, mb = _qlora(9), _qlora(9)
    pa = [p for p in ma.parameters() if p.requires_grad]
    pb = [p for p in mb.parameters() if p.requires_grad]
    assert len(pa) == 4 and all(p.dtype == torch.bfloat16 for p in pa)
    oa = bnb.optim.AdamW8bit(pa, lr=1e-3, capturable=True)
    ob = bnb.optim.AdamW8bit(pb, lr=1e-3)
    gen = torch.Generator(device="cpu").manual_seed(10)
    data = [(torch.randn(M, 1024, generator=gen).to(torch.bfloat16).cuda(),
             torch.randn(M, 512, generator=gen).to(torch.bfloat16).cuda()) for _ in range(7)]

    def train_step(model, opt, x, y):
        loss = torch.nn.functional.mse_loss(model(x), y)
        loss.backward()
        opt.step()
        return loss

    static_x, static_y = data[0][0].clone(), data[0][1].clone()
    losses_a, losses_b = [], []
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # two eager warm-up steps
        for x, y in data[:2]:
            oa.zero_grad(set_to_none=True)
            ob.zero_grad(set_to_none=True)
            static_x.copy_(x)
            static_y.copy_(y)
            losses_a.append(train_step(ma, oa, static_x, static_y).detach().float())
            losses_b.append(train_step(mb, ob, x, y).detach().float())
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    oa.zero_grad(set_to_none=True)
    with torch.cuda.graph(graph):
        static_loss = train_step(ma, oa, static_x, static_y)
    for x, y in data[2:]:
        static_x.copy_(x)
        static_y.copy_(y)
        graph.replay()
        losses_a.append(static_loss.detach().float().clone())
        ob.zero_grad(set_to_none=True)
        losses_b.append(train_step(mb, ob, x, y).detach().float())
    torch.cuda.synchronize()
    assert all(int(oa.state[p]["step"].item()) == 7 for p in pa) and all(ob.state[p]["step"] == 7 for p in pb)
    assert all(oa.state[p]["state1"].dtype == torch.uint8 for p in pa)
    torch.testing.assert_close(torch.stack(losses_a), torch.stack(losses_b), rtol=1.6e-2, atol=1e-5)
    for x, y in zip(pa, pb):
        torch.testing.assert_close(x, y)  # (bf16 tolerances)
    assert not torch.equal(ma[0].A, _qlora(9)[0].A), "the replays trained the adapters"
