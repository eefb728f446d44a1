"""CPU tests of the sequence-parallel LLM.int8() layers: the argument checks of the int32 scatter GEMM (against a fake
library), the rank-order destination list the fused row route hands it, and the layers' shape rules."""
import pytest
import torch

import bitsandbytes_b200.backends.cuda as cb
import bitsandbytes_b200.parallel as par
from bitsandbytes_b200.parallel import ColumnParallelLinear8bitLt, RowParallelLinear8bitLt, Shard8bit
from tests._parallel_sim import fake, simulate  # noqa: F401  (fake: a fixture)


def test_scatter_wrapper_checks(fake):
    """Bad destination counts, a row count that does not split over the destinations, a bad row stride, non-int8
    operands and non-int32 or too small destinations raise RuntimeError before any native call; a good call passes
    (n_outs, rows_per_out, M, N, K, ldc)."""
    CA, CB = torch.zeros(8, 64, dtype=torch.int8), torch.zeros(32, 64, dtype=torch.int8)

    def call(*, CA=CA, CB=CB, outs=None, ldc=32):
        outs = [torch.zeros(2, 32, dtype=torch.int32)] * 4 if outs is None else outs
        return cb.int8_gemm_partial_scatter(CA, CB, outs, ldc)

    bad = [({"outs": []}, "destinations"),
           ({"outs": [0x1000] * 9}, "destinations"),                                     # M = 8 over 9
           ({"CA": torch.zeros(16, 64, dtype=torch.int8), "outs": [0x1000] * 16}, "between 1 and 8"),
           ({"outs": [0x1000] * 3}, "do not split"),                                    # 8 % 3
           ({"ldc": 31}, "ldc"),
           ({"CA": torch.zeros(8, 64, dtype=torch.float16)}, "int8"),
           ({"CB": torch.zeros(32, 64, dtype=torch.int32)}, "int8"),
           ({"CB": torch.zeros(32, 48, dtype=torch.int8)}, "does not match"),
           ({"outs": [torch.zeros(2, 32)] * 4}, "int32"),
           ({"outs": [torch.zeros(2 * 32 - 1, dtype=torch.int32)] * 4}, "elements")]  # room for M/w rows only
    for kwargs, match in bad:
        with pytest.raises(RuntimeError, match=match):
            call(**kwargs)
    assert fake.calls == []
    assert call() and call(outs=[0x1000, 0x2000], ldc=40)
    assert call(outs=[torch.zeros(8, 32, dtype=torch.int32)])  # one destination: every row
    assert [n for n, _ in fake.calls] == ["cbnb_b200_int8_gemm_partial_scatter"] * 3
    # (CA, CB, outs, n_outs, rows_per_out, M, N, K, ldc, stream)
    assert [args[3:9] for _, args in fake.calls] == [(4, 2, 8, 32, 64, 32), (2, 4, 8, 32, 64, 40),
                                                     (1, 8, 8, 32, 64, 32)]
    assert fake.dests[1] == [0x1000, 0x2000]


def _simulated_world(monkeypatch, world, rank):
    """One rank of a simulated world: the statistics and codes of the row prologue and the reduction are CPU
    stand-ins."""
    simulate(monkeypatch, world, rank, [])
    monkeypatch.setattr(par, "int8_row_stats", lambda x, thr: (torch.ones(x.shape[0]), None))
    monkeypatch.setattr(par, "int8_quant_with_stats", lambda x, SCA, thr: torch.zeros(x.shape, dtype=torch.int8))
    monkeypatch.setattr(par, "int8_reduce_partials",
                        lambda parts, SCA, SCB, dtype, bias=None, *a, out=None: parts.sum(0).to(dtype))


def _k_shard(N=32, K=64, world=1, rank=0):
    kr = K // world
    return Shard8bit(CB=torch.zeros(N, kr, dtype=torch.int8), SCB=torch.ones(N), rows=N, row0=0, K=kr, k0=rank * kr)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_fused_row_route_scatters_in_rank_order(monkeypatch, fake, world):
    """For every rank of a simulated world, the fused SP row route hands the scatter GEMM slot r (this rank's) of every
    rank's [world, M/world, N] int32 buffer, in rank order, alternating between the two slots, and returns its tokens."""
    Ms, N, K = 2, 32, 48 * world
    for rank in range(world):
        _simulated_world(monkeypatch, world, rank)
        fake.dests.clear()
        layer = RowParallelLinear8bitLt(_k_shard(N, K, world, rank), K, sequence_parallel=True)
        peers = par.PeerPartials(Ms, N, "cpu", dtype=torch.int32)
        assert peers.bufs[0].shape == (world, Ms, N) and peers.bufs[0].dtype == torch.int32
        for step in range(3):
            y = par.fused_forward_row8_sp(layer, torch.zeros(world * Ms, K // world, dtype=torch.float16), peers)
            assert y.shape == (Ms, N)
            off = rank * Ms * N * 4
            assert fake.dests[step] == [(1 + (step & 1)) * 1_000_000 + s * 10_000 + off for s in range(world)]
        assert all(h.barriers == (2 if i == 0 else 1) for i, h in enumerate(peers.handles))


def _n_shard(N=32, K=64):
    return Shard8bit(CB=torch.zeros(N, K, dtype=torch.int8), SCB=torch.ones(N), rows=N, row0=0, K=K)


def test_column_layer_argument_rules():
    with pytest.raises(ValueError, match="gather_output=False"):
        ColumnParallelLinear8bitLt(_n_shard(), 32, sequence_parallel=True)
    with pytest.raises(ValueError, match="multiple of 16"):
        ColumnParallelLinear8bitLt(_n_shard(K=72), 32, gather_output=False, sequence_parallel=True)
    assert ColumnParallelLinear8bitLt(_n_shard(K=72), 32, gather_output=False).sequence_parallel is False
    assert ColumnParallelLinear8bitLt(_n_shard(), 32, gather_output=False, sequence_parallel=True).sequence_parallel
    with pytest.raises(ValueError, match="multiple of 16"):
        par.PeerInt8Input(8, 72, "cpu")


@pytest.mark.parametrize("shape,want", [((8, 64), (2, 32)), ((8, 3, 64), (2, 3, 32)), ((4, 5, 64), (1, 5, 32))])
def test_row_layer_sp_shapes(monkeypatch, fake, shape, want):
    """The row layer with SP returns this rank's share of the first dimension; the others keep their size.  The NCCL
    route computes the whole partial once (the broadcast form) and exchanges it."""
    _simulated_world(monkeypatch, 4, 1)
    layer = RowParallelLinear8bitLt(_k_shard(32, 256, 4, 1), 256, sequence_parallel=True)
    assert layer(torch.zeros(shape, dtype=torch.bfloat16)).shape == want
    assert [n for n, _ in fake.calls] == ["cbnb_b200_int8_gemm_multi_out"]


@pytest.mark.parametrize("shape", [(6, 64), (6, 4, 64), (3, 64)])
def test_row_layer_sp_needs_tokens_divisible_by_world(monkeypatch, fake, shape):
    _simulated_world(monkeypatch, 4, 1)
    layer = RowParallelLinear8bitLt(_k_shard(32, 256, 4, 1), 256, sequence_parallel=True)
    with pytest.raises(ValueError, match="world of 4"):
        layer(torch.zeros(shape, dtype=torch.bfloat16))
    assert fake.calls == []


@pytest.mark.parametrize("shape,want", [((2, 64), (8, 32)), ((2, 3, 64), (8, 3, 32)), ((1, 64), (4, 32))])
def test_column_layer_sp_shapes(monkeypatch, fake, shape, want):
    """The column layer with SP quantises only this rank's tokens and runs the GEMM on the gathered codes of all."""
    _simulated_world(monkeypatch, 4, 1)
    layer = ColumnParallelLinear8bitLt(_n_shard(), 128, gather_output=False, sequence_parallel=True)
    assert layer(torch.zeros(shape, dtype=torch.bfloat16)).shape == want
    names = [n for n, _ in fake.calls]
    assert names == ["cbnb_b200_int8_vector_quant_flags", "cbnb_b200_int8_gemm_multi_out"]
    tokens = shape[0] * (shape[1] if len(shape) == 3 else 1)
    assert fake.calls[0][1][5] == tokens                       # (A, out, rowStats, flags, threshold, rows, ...)
    assert fake.calls[1][1][10] == want[0] * (want[1] if len(want) == 3 else 1)  # M of the GEMM: all tokens
