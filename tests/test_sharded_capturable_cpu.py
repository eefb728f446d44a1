"""CPU tests of a capturable ``ShardedOptimizer`` (wrapping an optimizer made with ``capturable=True``), in a simulated
world (tests/_parallel_sim.py's collectives, the update and norm launches replaced by recorders): the update calls take
the device counters, one view per parameter into one counter tensor; every counter advances once per step, also for
parameters of which the rank holds no piece and for empty tensors; a tensor lr and the clip coefficient reach the call;
the refusals while capturing; the steps in state dicts and their in-place load."""
import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.optim.sharded as sh
from tests._parallel_sim import simulate

# two dtypes, 8-bit and 32-bit state, an empty tensor, and enough blocks that at w = 8 some rank holds no piece of a
# tensor
_SHAPES = [((64, 80), torch.float32), ((7,), torch.float32), ((0,), torch.float32), ((33, 33), torch.bfloat16),
           ((300,), torch.bfloat16), ((4096,), torch.bfloat16)]


def _model():
    torch.manual_seed(0)
    return [torch.nn.Parameter(torch.randn(*s).to(dt)) for s, dt in _SHAPES]


@pytest.fixture
def world(monkeypatch):
    """A simulated world of (w, r) on the CPU, which stands in for the CUDA device a capturable optimizer needs; every
    update launch is recorded with its steps, lr and coefficient, and the capture state is ``capturing["on"]``."""
    log, calls, capturing = [], [], {"on": False}

    def make(w, r):
        def launch(kind):
            def rec(name, g, p, s1, s2, *args, **kw):
                step, lr = (args[6], args[7]) if kind == "32" else (args[5], args[6])
                calls.append({"kind": kind, "steps": list(step), "lr": lr, "coef": kw.get("gnorm_scale_dev"),
                              "numels": [t.numel() for t in p]})
            return rec

        def norm(g, srcs, grad_local, grad_scale, norm_type, acc):
            log.append(("norm", acc.data_ptr()))

        def coef(values, norm_type, max_norm, out):
            out[0], out[1] = 2.0, 0.5

        simulate(monkeypatch, w, r, log)
        monkeypatch.setattr(sh, "_group_world_rank", lambda group: (w, r))
        monkeypatch.setattr(sh.dist, "broadcast", lambda t, src, group=None: None)
        monkeypatch.setattr(sh, "optimizer_update_32bit_multi_peers", launch("32"))
        monkeypatch.setattr(sh, "optimizer_update_8bit_blockwise_multi_peers", launch("8"))
        monkeypatch.setattr(sh, "optimizer_grad_norm_peers", norm)
        monkeypatch.setattr(sh, "optimizer_clip_coef", coef)
        monkeypatch.setattr(sh, "_capturing", lambda: capturing["on"])
        monkeypatch.setattr(sh, "_graph_device", lambda device: True)
        return calls, capturing

    return make


def _sharded(lr=1e-3, capturable=True, params=None):
    return sh.ShardedOptimizer(bnb.optim.AdamW8bit(_model() if params is None else params, lr=lr, min_8bit_size=1000,
                                                   capturable=capturable))


def _counter_index(opt, t):
    """The entry whose counter the one-element tensor t views (it must lie inside opt.steps)."""
    off = t.data_ptr() - opt.steps.data_ptr()
    assert t.dtype == torch.int32 and t.numel() == 1 and off % 4 == 0 and 0 <= off < 4 * opt.steps.numel()
    return off // 4


@pytest.mark.parametrize("w", [1, 2, 3, 8])
def test_calls_take_views_of_one_counter_tensor(world, w):
    for r in sorted({0, w // 2, w - 1}):
        calls, _ = world(w, r)
        opt = _sharded()
        assert opt.steps.dtype == torch.int32 and opt.steps.numel() == len(opt.entries) == len(_SHAPES)
        calls.clear()
        opt.step()
        seen = []
        for c in calls:
            for t in c["steps"]:
                seen.append(_counter_index(opt, t))
        assert sorted(seen) == sorted(e for _, e, _, _, _ in opt.pieces)   # each piece its own parameter's counter
        assert sum(sum(c["numels"]) for c in calls) == sum(n for *_, n, _ in opt.pieces)


@pytest.mark.parametrize("w", [1, 2, 3, 8])
def test_every_counter_advances_once_per_step(world, w):
    r = w - 1
    world(w, r)
    opt = _sharded()
    held = {e for _, e, _, _, _ in opt.pieces}
    if w == 8:
        assert len(held) < len(opt.entries)          # some parameter has no piece on this rank
    ptr = opt.steps.data_ptr()
    for k in range(1, 4):
        opt.step()
        assert opt.steps.tolist() == [k] * len(_SHAPES)      # the empty tensor and the pieces held elsewhere too
    assert opt.steps.data_ptr() == ptr
    non = _sharded(capturable=False)
    for _ in range(3):
        non.step()
    assert non.steps == [3] * len(_SHAPES)


def test_tensor_lr_is_passed_as_a_tensor_and_a_float_by_value(world):
    calls, _ = world(2, 0)
    lr = torch.full((1,), 1e-3)
    opt = _sharded(lr=lr)
    opt.step()
    assert calls and all(c["lr"] is lr for c in calls)
    lr.fill_(5e-4)                                    # a scheduler writing in place: the same tensor at the next step
    calls.clear()
    opt.step()
    assert all(c["lr"] is lr for c in calls)
    calls, _ = world(2, 0)
    calls.clear()
    opt = _sharded(lr=2e-3)
    opt.step()
    assert calls and all(c["lr"] == 2e-3 and not isinstance(c["lr"], torch.Tensor) for c in calls)


def test_clip_coefficient_reaches_the_calls_and_its_buffers_are_reused(world):
    calls, _ = world(3, 1)
    opt = _sharded()
    total = opt.clip_grad_norm_(1.0)
    opt.step()
    assert float(total) == 2.0
    coefs = {c["coef"].data_ptr() for c in calls}
    assert coefs == {total.data_ptr() + 4}
    calls.clear()
    total2 = opt.clip_grad_norm_(1.0)
    opt.step()
    assert total2.data_ptr() == total.data_ptr() and {c["coef"].data_ptr() for c in calls} == coefs
    calls.clear()
    opt.step()                                        # unclipped: no coefficient
    assert all(c["coef"] is None for c in calls)


def test_refusals_while_capturing(world):
    calls, capturing = world(2, 0)
    opt = _sharded()
    capturing["on"] = True
    with pytest.raises(RuntimeError, match="run one eager step"):           # no exchange buffer yet
        opt.step()
    with pytest.raises(RuntimeError, match="run one eager"):                # no clip buffers yet
        opt.clip_grad_norm_(1.0)
    capturing["on"] = False
    opt.clip_grad_norm_(1.0)
    opt.step()
    capturing["on"] = True
    calls.clear()
    opt.clip_grad_norm_(1.0)                                                 # warmed up: both can be captured
    opt.step()
    assert calls and all(c["coef"] is not None for c in calls)
    with pytest.raises(RuntimeError, match="error_if_nonfinite"):
        opt.clip_grad_norm_(1.0, error_if_nonfinite=True)
    for take in (opt.state_dict, opt.consolidated_state_dict):
        with pytest.raises(RuntimeError, match="captured"):
            take()
    plain = _sharded(capturable=False)
    calls.clear()
    with pytest.raises(RuntimeError, match="capturable=False"):
        plain.step()
    assert calls == []
    capturing["on"] = False
    assert opt.steps.tolist() == [2] * len(_SHAPES)   # (the recorders launch nothing: the captured add ran eagerly)


@pytest.mark.parametrize("w", [1, 3])
def test_state_dicts_round_trip_the_steps_in_place(world, w):
    world(w, w - 1)
    opt = _sharded()
    for _ in range(3):
        opt.step()
    sd = opt.state_dict()
    assert sd["steps"] == {i: 3 for i in range(len(_SHAPES))} and all(type(v) is int for v in sd["steps"].values())
    srcs = [sd]
    if w == 1:                                        # (the simulated world gathers no other shards)
        full = opt.consolidated_state_dict()
        assert [v["step"] for v in full["state"].values()] == [3] * len(_SHAPES)
        assert all(type(v["step"]) is int for v in full["state"].values())
        srcs.append(full)
    non = _sharded(capturable=False)
    for _ in range(3):
        non.step()
    assert non.state_dict()["steps"] == sd["steps"]
    other = _sharded()
    ptr = other.steps.data_ptr()
    state_ptrs = [{k: v.data_ptr() for k, v in st.items() if k in sh._STATE_KEYS} for *_, st in other.pieces]
    for src in srcs:
        other.steps.zero_()
        other.load_state_dict(src)
        assert other.steps.data_ptr() == ptr and other.steps.tolist() == [3] * len(_SHAPES)
        assert [{k: v.data_ptr() for k, v in st.items() if k in sh._STATE_KEYS} for *_, st in other.pieces] == \
            state_ptrs
        for (*_, a), (*_, b) in zip(opt.pieces, other.pieces):
            for k in sh._STATE_KEYS:
                if k in a:
                    assert torch.equal(a[k], b[k])
    non.load_state_dict(sd)
    assert non.steps == [3] * len(_SHAPES)


def test_refusals(world, monkeypatch):
    """What a capturable optimizer cannot shard: a trust ratio, AdEMAMix, parameters off a CUDA device."""
    world(2, 0)
    p = [torch.nn.Parameter(torch.randn(300))]
    for make in (lambda: bnb.optim.LAMB8bit(p, capturable=True), lambda: bnb.optim.AdEMAMix8bit(p, capturable=True)):
        with pytest.raises(ValueError):
            bnb.optim.ShardedOptimizer(make())
    assert bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(p, capturable=True)).capturable
    monkeypatch.undo()                                # the real device check: these parameters are on the CPU
    with pytest.raises(ValueError, match="CUDA device"):
        bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(p, capturable=True))
    assert not bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(p)).capturable
