"""CPU tests of ``bnb.optim.ShardedOptimizer``: the partition of the flat buffers, the per-tensor 8-bit / 32-bit
decision, the state bytes per rank, and, in a simulated world (collectives and the native launches replaced by
recorders), which collectives a step issues in which order with which bases; the refusals, the state-dict layouts, the
consolidation on one rank, and the gradient views."""
import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.optim.sharded as sh
from bitsandbytes_b200.optim.sharded import partition

# odd sizes, tensors smaller than one block, tensors spanning several ranks, an empty tensor
_NUMELS = [[1], [256], [257], [3, 5, 7], [1000, 1, 4096, 300], [100000, 17, 256 * 9 + 1], [0, 513, 0, 2]]


@pytest.mark.parametrize("numels", _NUMELS)
@pytest.mark.parametrize("world", range(1, 9))
def test_partition_owns_every_block_once(numels, world):
    starts, S, pieces = partition(numels, world)
    assert S % 256 == 0 and len(pieces) == world
    B = sum(-(-n // 256) for n in numels)
    assert world * S >= B * 256 > (world - 1) * S - 256 * world or B == 0
    owned = {}
    for r, mine in enumerate(pieces):
        for t, off, n in mine:
            assert off % 256 == 0 and 0 < n and off + n <= numels[t]          # block-aligned, never padding
            lo = starts[t] + off
            assert r * S <= lo and lo + n <= (r + 1) * S                       # inside rank r's equal shard
            assert n % 256 == 0 or off + n == numels[t]                        # whole blocks, or the real last block
            for e in range(lo, lo + n):
                assert e not in owned
                owned[e] = r
    real = {starts[t] + i for t, n in enumerate(numels) for i in range(n)}
    assert set(owned) == real
    for t in range(1, len(numels)):
        assert starts[t] == starts[t - 1] + 256 * -(-numels[t - 1] // 256)


@pytest.fixture
def world(monkeypatch):
    """A simulated world of (w, r): every collective and native launch is recorded."""
    log = []

    def make(w, r):
        def launch(kind):
            def rec(name, g, p, s1, s2, *args, **kw):
                srcs, dsts, gl, pl, scale = args[-5:]
                log.append((kind, name, [t.numel() for t in p], list(srcs), list(dsts), gl.data_ptr(), pl.data_ptr(),
                            scale))
            return rec

        monkeypatch.setattr(sh, "_group_world_rank", lambda group: (w, r))
        monkeypatch.setattr(sh.dist, "broadcast", lambda t, src, group=None: log.append(("broadcast", t.numel())))
        monkeypatch.setattr(sh.dist, "all_to_all_single",
                            lambda out, inp, group=None: log.append(("all_to_all", out.numel(), inp.numel())))
        monkeypatch.setattr(sh.dist, "all_gather_into_tensor",
                            lambda out, inp, group=None: log.append(("all_gather", out.data_ptr(), inp.data_ptr(),
                                                                     inp.numel())))
        monkeypatch.setattr(sh.dist, "gather_object",
                            lambda obj, out, dst=0, group=None: log.append(("gather", obj, out, dst)))
        monkeypatch.setattr(sh, "optimizer_update_32bit_multi_peers", launch("32"))
        monkeypatch.setattr(sh, "optimizer_update_8bit_blockwise_multi_peers", launch("8"))
        return log

    return make


def _model(dtype=torch.float32):
    torch.manual_seed(0)
    return [torch.nn.Parameter(torch.randn(*s).to(dtype)) for s in [(64, 80), (7,), (33, 33), (300,)]]


def test_state_is_8bit_by_whole_tensor_and_a_wth_of_the_bytes(world):
    """A tensor of 5120 elements has 8-bit state on every rank that holds a piece of it, however small the piece; the
    300- and 7-element tensors keep 32-bit state; the state bytes per rank are the unsharded bytes / w within a block
    per tensor edge."""
    for w in (1, 2, 3, 8):
        totals = []
        for r in range(w):
            world(w, r)
            params = _model()
            opt = bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(params, min_8bit_size=1000))
            for flat, e, s, n, st in opt.pieces:
                want = torch.uint8 if params[e].numel() >= 1000 else torch.float32
                assert st["state1"].dtype == want and st["state2"].dtype == want and st["state1"].numel() == n
                assert ("absmax1" in st) == (want == torch.uint8)
            totals.append(sum(v.numel() * v.element_size() for *_, st in opt.pieces for k, v in st.items()
                              if k in ("state1", "state2", "absmax1", "absmax2")))
        full = sum(2 * (p.numel() if p.numel() >= 1000 else 4 * p.numel()) + (8 * -(-p.numel() // 256)
                                                                           if p.numel() >= 1000 else 0)
                   for p in _model())
        assert sum(totals) == full
        slack = 2 * len(_model()) * 256 * 8
        assert all(t <= full / w + slack for t in totals), (w, totals, full)


def test_one_rank_exchanges_nothing(world):
    log = world(1, 0)
    params = _model(torch.bfloat16)
    opt = bnb.optim.ShardedOptimizer(bnb.optim.AdamW8bit(params, min_8bit_size=1000))
    log.clear()
    opt.step()
    flat = opt.flats[0]
    assert {e[0] for e in log} == {"8", "32"}
    for kind, name, numels, srcs, dsts, gl, pl, scale in log:
        assert srcs == [flat.grad.data_ptr()] and dsts == [flat.param.data_ptr()] and scale == 1.0
    assert sum(sum(e[2]) for e in log) == sum(p.numel() for p in params)


def test_step_issues_all_to_all_launches_all_gather(world):
    log = world(3, 2)
    params = _model(torch.float16)
    opt = bnb.optim.ShardedOptimizer(bnb.optim.Lion8bit(params, min_8bit_size=1000), grad_scale=1.0)
    log.clear()
    opt.step()
    kinds = [e[0] for e in log]
    assert kinds[0] == "all_to_all" and kinds[-1] == "all_gather" and kinds.count("all_to_all") == 1
    flat = opt.flats[0]
    S, es = flat.S, 2
    assert log[0][1:] == (3 * S, 3 * S)
    assert log[-1][1:] == (flat.param.data_ptr(), flat.param.data_ptr() + 2 * S * es, S)
    for kind, name, numels, srcs, dsts, gl, pl, scale in log[1:-1]:
        assert srcs == [flat.recv.data_ptr() + (r - 2) * S * es for r in range(3)]
        assert dsts == [flat.param.data_ptr()] and scale == 1.0


def test_refusals(world):
    world(2, 0)
    p = [torch.nn.Parameter(torch.randn(300))]
    for make in (lambda: bnb.optim.LAMB(p), lambda: bnb.optim.LARS(p, lr=0.1, momentum=0.9), lambda: bnb.optim.AdEMAMix8bit(p),
                 lambda: bnb.optim.PagedAdamW8bit(p), lambda: bnb.optim.Adam8bit(p, capturable=True)):
        with pytest.raises(ValueError):
            bnb.optim.ShardedOptimizer(make())
    with pytest.raises(ValueError):
        bnb.optim.ShardedOptimizer(torch.optim.SGD(p, lr=0.1))
    with pytest.raises(ValueError, match="one device"):
        bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(p + [torch.nn.Parameter(torch.zeros(4, device="meta"))]))
    opt = bnb.optim.Adam8bit(p)
    opt.state[p[0]]["step"] = 1
    with pytest.raises(ValueError, match="state"):
        bnb.optim.ShardedOptimizer(opt)


def test_grad_views_survive_zero_grad_and_none_counts_as_zeros(world):
    log = world(2, 0)
    params = _model()
    opt = bnb.optim.ShardedOptimizer(bnb.optim.SGD8bit(params, lr=0.1, momentum=0.9))
    flat = opt.flats[0]
    views = [p.grad for p in params]
    for p, s in zip(params, flat.starts):
        assert p.data.data_ptr() == flat.param.data_ptr() + 4 * s and p.grad.data_ptr() == flat.grad.data_ptr() + 4 * s
    params[0].grad.add_(2.0)
    assert flat.grad[:params[0].numel()].eq(2.0).all()
    opt.zero_grad()
    assert all(p.grad is v for p, v in zip(params, views)) and not flat.grad.any()
    params[1].grad = None
    params[2].grad = torch.full_like(params[2], 3.0)
    flat.grad[flat.starts[1]:flat.starts[1] + 7].fill_(5.0)
    opt.step()
    assert all(p.grad is v for p, v in zip(params, views))
    assert not flat.grad[flat.starts[1]:flat.starts[1] + 7].any()
    assert flat.grad[flat.starts[2]:flat.starts[2] + 33 * 33].eq(3.0).all()


def test_state_dict_layouts(world):
    """The shard lists its pieces with their partition; the consolidated dict has the unsharded optimizer's keys and
    shapes; loading the consolidated dict into another rank of another world slices that rank's blocks."""
    world(2, 1)
    params = _model()
    opt = bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(params, min_8bit_size=1000))
    for *_, st in opt.pieces:
        for k in ("state1", "state2", "absmax1", "absmax2"):
            if k in st:
                st[k].copy_(torch.arange(st[k].numel()).to(st[k].dtype))
    opt.steps = [3] * len(params)
    sd = opt.state_dict()
    assert sd["sharded"]["world"] == 2 and sd["sharded"]["rank"] == 1
    assert [(q["param"], q["offset"], q["numel"]) for q in sd["pieces"]] == \
        [(e, s - f.starts[f.index.index(e)], n) for f, e, s, n, _ in opt.pieces]
    opt.load_state_dict(sd)
    assert opt.steps == [3] * len(params)
    world(3, 0)
    opt3 = bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(_model(), min_8bit_size=1000))
    with pytest.raises(ValueError, match="partition"):
        opt3.load_state_dict(sd)
    # a world of one holds every piece: the consolidated dict is the unsharded optimizer's format
    world(1, 0)
    params1 = _model()
    opt1 = bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(params1, min_8bit_size=1000))
    for *_, st in opt1.pieces:
        for k in ("state1", "state2", "absmax1", "absmax2"):
            if k in st:
                st[k].copy_(torch.randint(0, 200, (st[k].numel(),)).to(st[k].dtype))
    opt1.steps = [5] * len(params1)
    full = opt1.consolidated_state_dict()
    key = bnb.optim.optimizer.Optimizer8bit._FSDP_WRAPPED_QUANT_STATE_KEY
    for k, v in full["state"].items():
        assert v["step"] == 5
        q = v[key]
        eight = params1[k].numel() >= 1000
        assert q["state1"].dtype == (torch.uint8 if eight else torch.float32) and q["state1"].shape == params1[k].shape
        assert ("absmax1" in q) == eight and ("qmap1" in q) == eight
        if eight:
            assert q["absmax2"].shape == (-(-params1[k].numel() // 256),)
    # ... and loads, sliced by blocks, into rank 1 of a world of 3
    world(3, 1)
    opt31 = bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(_model(), min_8bit_size=1000))
    opt31.load_state_dict(full)
    assert opt31.steps == [5] * len(params1)
    for f, e, s, n, st in opt31.pieces:
        off = s - f.starts[f.index.index(e)]
        q = full["state"][e][key]
        assert torch.equal(st["state1"], q["state1"].reshape(-1)[off:off + n])
        if "absmax1" in st:
            assert torch.equal(st["absmax1"], q["absmax1"][off // 256:off // 256 + -(-n // 256)])


def test_consolidation_gathers_to_one_rank_on_the_cpu(world, monkeypatch):
    """Rank 1 of 2 sends its shard to rank 0 and gets None; rank 0 assembles every tensor's state from both shards, on
    the CPU, in the unsharded layout."""
    key = bnb.optim.optimizer.Optimizer8bit._FSDP_WRAPPED_QUANT_STATE_KEY
    opts = []
    for r in range(2):
        log = world(2, r)
        opt = bnb.optim.ShardedOptimizer(bnb.optim.Adam8bit(_model(), min_8bit_size=1000))
        g = torch.Generator().manual_seed(r)
        for *_, st in opt.pieces:
            for k in ("state1", "state2", "absmax1", "absmax2"):
                if k in st:
                    st[k].copy_(torch.randint(0, 200, (st[k].numel(),), generator=g).to(st[k].dtype))
        opts.append(opt)
    log.clear()
    assert opts[1].consolidated_state_dict() is None
    (_, shard1, out, dst), = log
    assert out is None and dst == 0
    monkeypatch.setattr(sh.dist, "gather_object", lambda obj, out, dst=0, group=None: out.__setitem__(
        slice(None), [obj, shard1]))
    full = opts[0].consolidated_state_dict()
    params = _model()
    for opt in opts:
        for f, e, s, n, st in opt.pieces:
            off = s - f.starts[f.index.index(e)]
            q = full["state"][e][key]
            assert q["state1"].device.type == "cpu" and q["state1"].shape == params[e].shape
            assert torch.equal(q["state1"].reshape(-1)[off:off + n], st["state1"])
            if "absmax2" in st:
                assert torch.equal(q["absmax2"][off // 256:off // 256 + -(-n // 256)], st["absmax2"])
