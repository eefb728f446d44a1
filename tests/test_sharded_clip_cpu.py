"""CPU tests of ``ShardedOptimizer.clip_grad_norm_``: in a simulated world (collectives and native launches replaced by
recorders), which collectives and launches a clipped step issues, in which order and with which addresses; that a step
without clipping issues exactly the calls of the unclipped step; and the refusals."""
import math

import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.optim.sharded as sh


@pytest.fixture
def world(monkeypatch):
    """A simulated world of (w, r): every collective and native launch is recorded; the clip coefficient launch writes
    the norm ``norm_value`` and the coefficient 0.5."""
    log = []
    state = {"norm": 3.0}

    def make(w, r):
        def launch(kind):
            def rec(name, g, p, s1, s2, *args, **kw):
                srcs, dsts, gl, pl, scale = args[-5:]
                coef = kw.get("gnorm_scale_dev")
                log.append((kind, name, [t.numel() for t in p], list(srcs), list(dsts), gl.data_ptr(), pl.data_ptr(),
                            scale, sorted(kw), None if coef is None else coef.data_ptr()))
            return rec

        def norm(g, srcs, grad_local, grad_scale, norm_type, acc):
            log.append(("norm", [t.numel() for t in g], list(srcs), grad_local.data_ptr(), grad_scale, norm_type,
                        acc.data_ptr(), acc.dtype, acc.numel()))

        def coef(values, norm_type, max_norm, out):
            log.append(("coef", values.data_ptr(), values.numel(), values.dtype, norm_type, max_norm, out.data_ptr()))
            out[0], out[1] = state["norm"], 0.5

        monkeypatch.setattr(sh, "_group_world_rank", lambda group: (w, r))
        monkeypatch.setattr(sh.dist, "broadcast", lambda t, src, group=None: log.append(("broadcast", t.numel())))
        monkeypatch.setattr(sh.dist, "all_to_all_single",
                            lambda out, inp, group=None: log.append(("all_to_all", out.numel(), inp.numel())))
        monkeypatch.setattr(sh.dist, "all_gather_into_tensor",
                            lambda out, inp, group=None: log.append(("all_gather", out.data_ptr(), inp.data_ptr(),
                                                                     inp.numel(), out.dtype)))
        monkeypatch.setattr(sh, "optimizer_update_32bit_multi_peers", launch("32"))
        monkeypatch.setattr(sh, "optimizer_update_8bit_blockwise_multi_peers", launch("8"))
        monkeypatch.setattr(sh, "optimizer_grad_norm_peers", norm)
        monkeypatch.setattr(sh, "optimizer_clip_coef", coef)
        return log, state

    return make


def _model():
    """Two dtypes (two flat buffers), tensors with 8-bit and with 32-bit state."""
    torch.manual_seed(0)
    shapes = [((64, 80), torch.float32), ((7,), torch.float32), ((33, 33), torch.bfloat16), ((300,), torch.bfloat16),
              ((4096,), torch.bfloat16)]
    return [torch.nn.Parameter(torch.randn(*s).to(dt)) for s, dt in shapes]


def _srcs(opt, f):
    if opt.world == 1:
        return [f.grad.data_ptr()]
    es, s0 = f.grad.element_size(), opt.rank * f.S
    return [f.recv.data_ptr() + (r * f.S - s0) * es for r in range(opt.world)]


@pytest.mark.parametrize("norm_type", [2.0, math.inf])
@pytest.mark.parametrize("w", [1, 2, 3, 8])
def test_clip_then_step_issues_exchange_norm_gather_coef_scaled_updates(world, w, norm_type):
    for r in sorted({0, w - 1}):
        log, _ = world(w, r)
        opt = sh.ShardedOptimizer(bnb.optim.AdamW8bit(_model(), min_8bit_size=1000))
        log.clear()
        total = opt.clip_grad_norm_(1.0, norm_type=norm_type)
        assert total.dim() == 0 and total.dtype == torch.float32 and float(total) == 3.0
        k = 0
        if w > 1:                                                      # the step's exchange, done now, one per flat
            for f in opt.flats:
                assert log[k] == ("all_to_all", w * f.S, w * f.S)
                k += 1
        acc = None
        for f in opt.flats:                                            # the norm over this rank's pieces of each flat
            numels = [n for flat, _, _, n, _ in opt.pieces if flat is f]
            kind, got, srcs, gl, scale, nt, acc_ptr, acc_dtype, acc_n = log[k]
            assert kind == "norm" and got == numels and srcs == _srcs(opt, f) and gl == f.grad.data_ptr()
            assert scale == 1.0 / w and nt == norm_type and acc_dtype == torch.float64 and acc_n == 1
            assert acc is None or acc_ptr == acc                       # one accumulator for every flat
            acc = acc_ptr
            k += 1
        if w > 1:                                                      # one fp64 value per rank
            kind, out, inp, n, dtype = log[k]
            assert kind == "all_gather" and inp == acc and n == 1 and dtype == torch.float64
            values = out
            k += 1
        else:
            values = acc
        kind, vptr, vn, vdtype, nt, max_norm, out = log[k]
        assert (kind, vptr, vn, vdtype, nt, max_norm) == ("coef", values, w, torch.float64, norm_type, 1.0)
        assert total.data_ptr() == out
        assert len(log) == k + 1
        log.clear()
        opt.step()
        kinds = [e[0] for e in log]
        assert "all_to_all" not in kinds and "norm" not in kinds and "coef" not in kinds
        launches = [e for e in log if e[0] in ("8", "32")]
        assert launches and kinds[:len(launches)] == [e[0] for e in launches]
        for e in launches:
            f = next(f for f in opt.flats if f.grad.data_ptr() == e[5])
            assert e[3] == _srcs(opt, f) and e[4] == [f.param.data_ptr()]
            assert e[8] == ["gnorm_scale_dev", "skip_zeros"] and e[9] == out + 4     # the coefficient's address
        assert sum(sum(e[2]) for e in launches) == sum(n for *_, n, _ in opt.pieces)
        gathers = log[len(launches):]
        if w == 1:
            assert gathers == []
        else:
            assert [(e[0], e[1], e[3]) for e in gathers] == [("all_gather", f.param.data_ptr(), f.S)
                                                             for f in opt.flats]


def _step_log(world, w, r, clip_first):
    log, _ = world(w, r)
    opt = sh.ShardedOptimizer(bnb.optim.Lion8bit(_model(), min_8bit_size=1000))
    if clip_first:                                     # a clipped step first: the next one must be the plain one again
        opt.clip_grad_norm_(0.5)
        opt.step()
    log.clear()
    opt.step()
    return opt, list(log)


@pytest.mark.parametrize("w", [1, 3])
def test_step_without_clip_issues_the_unclipped_calls(world, w):
    """The calls of a plain step: all-to-all per flat, the unscaled entries with the arguments of before (no
    gnorm_scale_dev), the parameter all-gathers; also after a clipped step."""
    for clip_first in (False, True):
        opt, log = _step_log(world, w, w - 1, clip_first)
        k = 0
        if w > 1:
            assert log[:len(opt.flats)] == [("all_to_all", w * f.S, w * f.S) for f in opt.flats]
            k = len(opt.flats)
        launches = [e for e in log[k:] if e[0] in ("8", "32")]
        assert log[k:k + len(launches)] == launches
        for e in launches:
            f = next(f for f in opt.flats if f.grad.data_ptr() == e[5])
            assert e[3] == _srcs(opt, f) and e[4] == [f.param.data_ptr()] and e[7] == 1.0 / w
            assert e[8] == ["skip_zeros"] and e[9] is None
        rest = log[k + len(launches):]
        assert [(e[0], e[1], e[2], e[3]) for e in rest] == (
            [] if w == 1 else [("all_gather", f.param.data_ptr(), f.param.data_ptr() + (w - 1) * f.S *
                                f.param.element_size(), f.S) for f in opt.flats])


def test_refusals(world):
    world(2, 1)
    opt = sh.ShardedOptimizer(bnb.optim.Adam8bit(_model(), min_8bit_size=1000))
    for bad in (1, 1.0, 3, 0, -math.inf, "fro"):
        with pytest.raises(ValueError, match="norm_type"):
            opt.clip_grad_norm_(1.0, norm_type=bad)
    opt.clip_grad_norm_(1.0)
    with pytest.raises(RuntimeError, match="already"):
        opt.clip_grad_norm_(1.0)
    with pytest.raises(RuntimeError, match="closure"):
        opt.step(lambda: 0.0)
    opt.step()
    opt.clip_grad_norm_(1.0)                       # one clip per step
    opt.step()


def test_nonfinite_norm_raises_only_when_asked_and_the_step_exchanges_again(world):
    log, state = world(2, 0)
    opt = sh.ShardedOptimizer(bnb.optim.Adam8bit(_model(), min_8bit_size=1000))
    state["norm"] = math.inf
    assert math.isinf(float(opt.clip_grad_norm_(1.0)))
    opt.step()
    log.clear()
    with pytest.raises(RuntimeError, match="non-finite"):
        opt.clip_grad_norm_(1.0, error_if_nonfinite=True)
    log.clear()
    opt.step()                                     # not clipped: the step exchanges the gradients itself
    assert [e[0] for e in log].count("all_to_all") == len(opt.flats)
    assert all(e[9] is None for e in log if e[0] in ("8", "32"))
    state["norm"] = 2.0
    assert float(opt.clip_grad_norm_(1.0, error_if_nonfinite=True)) == 2.0


def test_none_gradient_counts_as_zeros(world):
    world(2, 0)
    params = _model()
    opt = sh.ShardedOptimizer(bnb.optim.Adam8bit(params, min_8bit_size=1000))
    flat = next(f for f in opt.flats if f.dtype == torch.bfloat16)
    views = [p.grad for p in params]
    flat.grad.fill_(1.0)
    params[2].grad = None
    params[3].grad = torch.full_like(params[3], 2.0)
    opt.clip_grad_norm_(1.0)
    assert all(p.grad is v for p, v in zip(params, views))
    s2, s3 = (flat.starts[next(i for i, q in enumerate(flat.params) if q is params[k])] for k in (2, 3))
    assert not flat.grad[s2:s2 + params[2].numel()].any()
    assert flat.grad[s3:s3 + 300].eq(2.0).all()
