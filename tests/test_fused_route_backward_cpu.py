"""CPU tests of the backward of the symmetric-memory routes (``grad_peers``), in a simulated world of 4 seen from rank 1:
which peer copies, barriers and ``reduce_partials_ptrs`` calls each route's backward issues, with which row windows and
pointer order; that no NCCL collective runs; the ``grad_peers`` checks; and the refusal without ``grad_peers``.  Each
route runs its layer's own forward (``layer._forward(x, peers, sp)``), replaced here by zeros of the output shape."""
import pytest
import torch

import bitsandbytes_b200.parallel as par
from bitsandbytes_b200.parallel import (ColumnParallelLinear4bit, ColumnParallelLinear8bitLt, RowParallelLinear4bit,
                                        RowParallelLinear8bitLt, Shard4bit, Shard8bit)
from tests._parallel_sim import peer_ptrs, simulate

WORLD, RANK = 4, 1
M, K, N = 8, 128, 256   # tokens, in_features, out_features of the column layer (the row layer: N -> K)
BF = torch.bfloat16


def _shard4(rows, K_, row0=0, k0=0):
    return Shard4bit(packed=torch.zeros(rows * K_ // 2, dtype=torch.uint8), absmax=torch.ones(rows * K_ // 64),
                     absmax_8bit=None, absmax_code=None, absmax_offset=None, rows=rows, row0=row0, K=K_, blocksize=64,
                     quant_type="nf4", k0=k0)


def _shard8(rows, K_, row0=0, k0=0):
    return Shard8bit(CB=torch.zeros(rows, K_, dtype=torch.int8), SCB=torch.ones(rows), rows=rows, row0=row0, K=K_,
                     k0=k0)


@pytest.fixture
def world4(monkeypatch):
    """Rank 1 of 4: every NCCL collective fails the test, the forward bodies return zeros, the products are zeros and
    ``reduce_partials_ptrs`` records its arguments."""
    log = []

    def no_collective(*args, **kwargs):
        raise AssertionError("an NCCL collective ran in the fused backward")

    def reduce_ptrs(ptrs, M_, N_, dtype, row0=0, rows=None, bias=None, out=None):
        rows = M_ - row0 if rows is None else rows
        log.append(("reduce", list(ptrs), M_, N_, dtype, row0, rows))
        return torch.zeros(rows, N_, dtype=dtype)

    simulate(monkeypatch, WORLD, RANK, log)
    for name in ("all_gather_into_tensor", "all_to_all_single", "all_reduce"):
        monkeypatch.setattr(par.dist, name, no_collective)
    monkeypatch.setattr(par, "reduce_partials", no_collective)
    monkeypatch.setattr(par, "reduce_partials_ptrs", reduce_ptrs)
    monkeypatch.setattr(par, "input_grad_dequant_matmul",
                        lambda G, shard, dtype: torch.zeros(G.shape[0], shard.K, dtype=dtype))
    return log, monkeypatch


def _peer_grad(M_, F_, dtype):
    return par.PeerInputGrad(M_, F_, dtype, "cpu")


def _column(kind, sp):
    shard = _shard4(N // WORLD, K, row0=RANK * N // WORLD) if kind == "4bit" else _shard8(N // WORLD, K,
                                                                                         row0=RANK * N // WORLD)
    cls = ColumnParallelLinear4bit if kind == "4bit" else ColumnParallelLinear8bitLt
    return cls(shard, N, gather_output=not sp, sequence_parallel=sp)


def _row(kind, sp, input_is_parallel=True):
    shard = (_shard4 if kind == "4bit" else _shard8)(K, N // WORLD, k0=RANK * N // WORLD)
    cls = RowParallelLinear4bit if kind == "4bit" else RowParallelLinear8bitLt
    return cls(shard, N, input_is_parallel=input_is_parallel, sequence_parallel=sp)


def _route(monkeypatch, kind, family, layer):
    """The route function of a family, the layer's forward replaced by zeros of the output shape."""
    out = {"col": lambda x: torch.zeros(M, N, dtype=x.dtype),
           "col_sp": lambda x: torch.zeros(M, N // WORLD, dtype=x.dtype),
           "row": lambda x: torch.zeros(M, K, dtype=x.dtype),
           "row_sp": lambda x: torch.zeros(M // WORLD, K, dtype=x.dtype)}[family]
    monkeypatch.setattr(layer, "_forward", lambda x, peers=None, sp=None: out(x))
    if kind == "4bit":
        name = {"col": "fused_forward", "col_sp": "fused_forward_col_sp", "row": "fused_forward_row",
                "row_sp": "fused_forward_row_sp"}[family]
    else:
        name = {"col": "fused_forward_col8", "col_sp": "fused_forward_col8_sp", "row": "fused_forward_row8",
                "row_sp": "fused_forward_row8_sp"}[family]
    return getattr(par, name)


KINDS = ["4bit", "int8"]


@pytest.mark.parametrize("kind", KINDS)
def test_column_backward_pulls_every_partial(world4, kind):
    """Column layer: the partial into this rank's own slot, one barrier, one reduction over all M rows of the four
    ranks' slots in rank order; the next backward takes the other slot.  No copy, no collective."""
    log, mp = world4
    layer = _column(kind, sp=False)
    fn = _route(mp, kind, "col", layer)
    gp = _peer_grad(M, K, torch.float32)
    log.clear()
    for step in range(2):
        x = torch.zeros(M, K, dtype=BF, requires_grad=True)
        fn(layer, x, None, grad_peers=gp).sum().backward()
        assert x.grad.shape == (M, K) and x.grad.dtype == BF
        assert log[-2:] == [("barrier", step), ("reduce", peer_ptrs(step, WORLD), M, K, BF, 0, M)]
    assert len(log) == 4


@pytest.mark.parametrize("kind", KINDS)
def test_sequence_parallel_column_backward_reduces_its_own_rows(world4, kind):
    """SP column layer: the same partial over all M tokens, and this rank reduces only its tokens' rows
    [rank*M/w, (rank+1)*M/w) -- the reduce-scatter by pull."""
    log, mp = world4
    layer = _column(kind, sp=True)
    fn = _route(mp, kind, "col_sp", layer)
    x = torch.zeros(M // WORLD, K, dtype=BF, requires_grad=True)
    gp = _peer_grad(M, K, torch.float32)
    log.clear()
    fn(layer, x, None, grad_peers=gp).sum().backward()
    assert x.grad.shape == (M // WORLD, K)
    assert log == [("barrier", 0), ("reduce", peer_ptrs(0, WORLD), M, K, BF, RANK * M // WORLD, M // WORLD)]


@pytest.mark.parametrize("kind", KINDS)
def test_sequence_parallel_row_backward_gathers_grad_rows(world4, kind):
    """SP row layer: this rank's token rows of grad_y copied into its rows of every rank's [M, N] slot, in rank order,
    one barrier, then the local product; no reduction."""
    log, mp = world4
    layer = _row(kind, sp=True)
    fn = _route(mp, kind, "row_sp", layer)
    x = torch.zeros(M, N // WORLD, dtype=BF, requires_grad=True)
    gp = _peer_grad(M, K, BF)
    log.clear()
    fn(layer, x, None, grad_peers=gp).sum().backward()
    assert x.grad.shape == (M, N // WORLD)
    Ms = M // WORLD
    assert log == [("copy", 0, r, (Ms, K), BF, RANK * Ms * K) for r in range(WORLD)] + [("barrier", 0)]


@pytest.mark.parametrize("kind", KINDS)
def test_row_backward_with_the_whole_input_gathers_columns(world4, kind):
    """input_is_parallel=False: this rank's gradient columns copied into every rank's [M, in_features] slot, one
    barrier; the gradient is the whole input's."""
    log, mp = world4
    layer = _row(kind, sp=False, input_is_parallel=False)
    fn = _route(mp, kind, "row", layer)
    x = torch.zeros(M, N, dtype=BF, requires_grad=True)
    gp = _peer_grad(M, N, BF)
    log.clear()
    fn(layer, x, None, grad_peers=gp).sum().backward()
    assert x.grad.shape == (M, N)
    assert log == [("copy", 0, r, (M, N), BF, 0) for r in range(WORLD)] + [("barrier", 0)]


@pytest.mark.parametrize("kind", KINDS)
def test_row_backward_with_parallel_input_exchanges_nothing(world4, kind):
    log, mp = world4
    layer = _row(kind, sp=False)
    fn = _route(mp, kind, "row", layer)
    x = torch.zeros(M, N // WORLD, dtype=BF, requires_grad=True)
    log.clear()
    fn(layer, x, None, grad_peers=_peer_grad(3, 5, torch.float16)).sum().backward()  # only the group is checked
    assert x.grad.shape == (M, N // WORLD) and log == []


@pytest.mark.parametrize("kind", KINDS)
def test_grad_peers_mismatches_raise(world4, kind):
    """A PeerInputGrad of another token count, width or dtype, or something else altogether, raises ValueError at the
    forward, before anything runs."""
    log, mp = world4
    col, col_sp = _column(kind, sp=False), _column(kind, sp=True)
    row_sp, row_full = _row(kind, sp=True), _row(kind, sp=False, input_is_parallel=False)
    cases = [(_route(mp, kind, "col", col), col, (M, K), [(M, K, BF), (M // 2, K, torch.float32),
                                                          (M, K // 2, torch.float32)]),
             (_route(mp, kind, "col_sp", col_sp), col_sp, (M // WORLD, K), [(M // WORLD, K, torch.float32),
                                                                            (M, K, BF)]),
             (_route(mp, kind, "row_sp", row_sp), row_sp, (M, N // WORLD), [(M, N // WORLD, BF), (M, K, torch.float16),
                                                                           (M // WORLD, K, BF)]),
             (_route(mp, kind, "row", row_full), row_full, (M, N), [(M, K, BF), (M, N, torch.float32)])]
    log.clear()
    for fn, layer, xshape, bad in cases:
        for shape in bad:
            x = torch.zeros(xshape, dtype=BF, requires_grad=True)
            with pytest.raises(ValueError, match="PeerInputGrad"):
                fn(layer, x, None, grad_peers=_peer_grad(*shape))
        with pytest.raises(ValueError, match="PeerInputGrad"):
            fn(layer, torch.zeros(xshape, dtype=BF, requires_grad=True), None, grad_peers=object())
    assert [e for e in log if e[0] != "copy"] == []


def test_grad_peers_of_another_group_raise(world4):
    log, mp = world4
    layer = _row("4bit", sp=False)
    fn = _route(mp, "4bit", "row", layer)
    gp = _peer_grad(M, K, BF)
    gp.group = object()
    with pytest.raises(ValueError, match="process group"):
        fn(layer, torch.zeros(M, N // WORLD, dtype=BF, requires_grad=True), None, grad_peers=gp)


def test_sp_row_layer_with_the_whole_input_needs_one_slot_shape(world4):
    """SP with input_is_parallel=False exchanges [M, N] and [M, in_features]: refused unless they agree."""
    log, mp = world4
    layer = _row("4bit", sp=True, input_is_parallel=False)
    fn = _route(mp, "4bit", "row_sp", layer)
    with pytest.raises(ValueError, match="input_is_parallel=False"):
        fn(layer, torch.zeros(M, N, dtype=BF, requires_grad=True), None, grad_peers=_peer_grad(M, K, BF))


@pytest.mark.parametrize("kind", KINDS)
def test_without_grad_peers_the_routes_stay_inference_only(world4, kind):
    """A grad-requiring input without grad_peers is refused; under no_grad, or with an input that needs no grad, the
    forward body runs as it is and no backward is attached."""
    log, mp = world4
    col, col_sp, row, row_sp = _column(kind, False), _column(kind, True), _row(kind, False), _row(kind, True)
    for family, layer, xshape in [("col", col, (M, K)), ("col_sp", col_sp, (M // WORLD, K)),
                                  ("row", row, (M, N // WORLD)), ("row_sp", row_sp, (M, N // WORLD))]:
        fn = _route(mp, kind, family, layer)
        x = torch.zeros(xshape, dtype=BF, requires_grad=True)
        with pytest.raises(RuntimeError, match="inference only"):
            fn(layer, x, None)
        with torch.no_grad():
            assert fn(layer, x, None, grad_peers=_peer_grad(M, K, torch.float32)).grad_fn is None
        assert fn(layer, x.detach(), None).grad_fn is None
    assert log == []


@pytest.mark.parametrize("kind", KINDS)
def test_training_call_does_not_return_the_output_slot(world4, kind):
    """The gathered column route returns its PeerGather slot; a training call returns a copy, which autograd may keep
    past the slot's next use, and the row route's whole-input gradient is a copy of its PeerInputGrad slot."""
    log, mp = world4
    layer = _column(kind, sp=False)
    slot = torch.zeros(M, N, dtype=BF)
    mp.setattr(layer, "_forward", lambda x, peers=None, sp=None: slot)
    fn = par.fused_forward if kind == "4bit" else par.fused_forward_col8
    x = torch.zeros(M, K, dtype=BF, requires_grad=True)
    assert fn(layer, x.detach(), None) is slot
    y = fn(layer, x, None, grad_peers=_peer_grad(M, K, torch.float32))
    assert y.data_ptr() != slot.data_ptr() and torch.equal(y, slot)
    row = _row(kind, sp=False, input_is_parallel=False)
    rfn = _route(mp, kind, "row", row)
    gp = _peer_grad(M, N, BF)
    xr = torch.zeros(M, N, dtype=BF, requires_grad=True)
    rfn(row, xr, None, grad_peers=gp).sum().backward()
    assert all(xr.grad.data_ptr() != b.data_ptr() for b in gp.bufs)
