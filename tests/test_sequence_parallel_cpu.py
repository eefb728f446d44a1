"""CPU tests of the sequence-parallel Linear4bit layers: the argument checks of the scatter partial GEMM (against a fake
library), the rank-order destination list of its symmetric-memory slots, and the layers' shape rules."""
import pytest
import torch

import bitsandbytes_b200.backends.cuda as cb
import bitsandbytes_b200.parallel as par
from bitsandbytes_b200.parallel import ColumnParallelLinear4bit, RowParallelLinear4bit, Shard4bit
from tests._parallel_sim import fake, simulate  # noqa: F401  (fake: a fixture)


def _gemm4_args(M=8, N=32, K=64, dtype=torch.bfloat16):
    """(A, B, shapeB, absmax, blocksize, quant_type) of an NF4 weight [N, K], blocksize 64."""
    return (torch.zeros(M, K, dtype=dtype), torch.zeros(N * K // 2, dtype=torch.uint8), (N, K),
            torch.ones(N * K // 64), 64, "nf4")


def test_scatter_wrapper_checks(fake):
    """Bad destination counts, a row count that does not split over the destinations, a bad activation dtype and
    non-fp32 or too small destinations raise RuntimeError before any native call; a good call passes rows_per_out."""
    A, B, shapeB, absmax, bs, qt = _gemm4_args()

    def call(*, A=A, outs=None, ldc=32):
        outs = [torch.zeros(2, 32)] * 4 if outs is None else outs
        return cb.gemm_4bit_partial_scatter(A, B, shapeB, absmax, bs, qt, None, None, None, outs, ldc)

    bad = [({"outs": []}, "destinations"),
           ({"outs": [0x1000] * 9}, "destinations"),                           # M = 8 over 9 destinations
           ({"A": torch.zeros(16, 64, dtype=torch.bfloat16), "outs": [0x1000] * 16}, "between 1 and 8"),
           ({"outs": [0x1000] * 3}, "do not split"),                          # 8 % 3
           ({"A": torch.zeros(8, 64, dtype=torch.int32)}, "dtype"),
           ({"outs": [torch.zeros(2, 32, dtype=torch.bfloat16)] * 4}, "float32"),
           ({"outs": [torch.zeros(2 * 32 - 1)] * 4}, "elements"),             # room for M/w rows, not more
           ({"ldc": 31}, "ldc")]
    for kwargs, match in bad:
        with pytest.raises(RuntimeError, match=match):
            call(**kwargs)
    assert fake.calls == []
    assert call() and call(outs=[0x1000, 0x2000], ldc=40)
    assert call(outs=[torch.zeros(8, 32)])  # one destination: every row
    names = [n for n, _ in fake.calls]
    assert names == ["cbnb_b200_gemm_4bit_partial_scatter"] * 3
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, outs, n_outs, rows_per_out, M, N, K, ldc, ...)
    assert [args[7:13] for _, args in fake.calls] == [(4, 2, 8, 32, 64, 32), (2, 4, 8, 32, 64, 40),
                                                     (1, 8, 8, 32, 64, 32)]


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_scatter_destinations_are_in_rank_order(monkeypatch, world):
    """For every rank of a simulated world, the scatter list of a [world, M/world, N] slot is slot r (this rank's) of
    every rank's buffer, in rank order, and successive steps alternate between the two slots."""
    Ms, N = 4, 16
    for rank in range(world):
        simulate(monkeypatch, world, rank, [])
        peers = par.PeerPartials(Ms, N, "cpu")
        assert peers.bufs[0].shape == (world, Ms, N)
        for step in range(3):
            local, bases, _ = peers.slot()
            assert local is peers.bufs[step & 1]
            off = rank * Ms * N * 4
            assert peers.scatter_ptrs(bases, off) == [(1 + (step & 1)) * 1_000_000 + s * 10_000 + off
                                                      for s in range(world)]


def _shard(N=32, K=64, k0=0):
    return Shard4bit(packed=torch.zeros(N * K // 2, dtype=torch.uint8), absmax=torch.ones(N * K // 64),
                     absmax_8bit=None, absmax_code=None, absmax_offset=None, rows=N, row0=0, K=K, blocksize=64,
                     quant_type="nf4", k0=k0)


def test_column_layer_rejects_sp_with_gathered_output():
    with pytest.raises(ValueError, match="gather_output=False"):
        ColumnParallelLinear4bit(_shard(), 32, sequence_parallel=True)
    assert ColumnParallelLinear4bit(_shard(), 32, gather_output=False, sequence_parallel=True).sequence_parallel


@pytest.fixture
def world4(monkeypatch, fake):
    """A simulated world of 4 on the CPU: the collectives only check their shapes, the reduction sums on the CPU."""
    simulate(monkeypatch, 4, 1, [])
    monkeypatch.setattr(par, "reduce_partials", lambda parts, dtype, bias=None: parts.sum(0).to(dtype))
    return fake


@pytest.mark.parametrize("shape,want", [((8, 64), (2, 32)), ((8, 3, 64), (2, 3, 32)), ((4, 5, 64), (1, 5, 32))])
def test_row_layer_sp_shapes(world4, shape, want):
    """The row layer with SP returns this rank's share of the first dimension; the others keep their size."""
    layer = RowParallelLinear4bit(_shard(), 256, sequence_parallel=True)
    assert layer(torch.zeros(shape, dtype=torch.bfloat16)).shape == want
    assert [n for n, _ in world4.calls] == ["cbnb_b200_gemm_4bit_partial"]


@pytest.mark.parametrize("shape", [(6, 64), (6, 4, 64), (3, 64)])
def test_row_layer_sp_needs_tokens_divisible_by_world(world4, shape):
    layer = RowParallelLinear4bit(_shard(), 256, sequence_parallel=True)
    with pytest.raises(ValueError, match="world of 4"):
        layer(torch.zeros(shape, dtype=torch.bfloat16))
    assert world4.calls == []


@pytest.mark.parametrize("shape,want", [((2, 64), (8, 32)), ((2, 3, 64), (8, 3, 32)), ((1, 64), (4, 32))])
def test_column_layer_sp_shapes(world4, shape, want):
    """The column layer with SP gathers the ranks' tokens along the first dimension."""
    layer = ColumnParallelLinear4bit(_shard(), 128, gather_output=False, sequence_parallel=True)
    assert layer(torch.zeros(shape, dtype=torch.bfloat16)).shape == want
    assert [n for n, _ in world4.calls] == ["cbnb_b200_gemm_4bit_strided"]
    assert world4.calls[0][1][8] == want[0] * (want[1] if len(want) == 3 else 1)  # M of the GEMM: all tokens
