"""CPU tests of the tensor-parallel Linear4bit backward: the refusal of grad-requiring input by the symmetric-memory
routes, and the collectives the backward runs in a simulated world of 4."""
import pytest
import torch

import bitsandbytes_b200.parallel as par
from bitsandbytes_b200.parallel import ColumnParallelLinear4bit, RowParallelLinear4bit, Shard4bit
from tests._parallel_sim import fake, simulate  # noqa: F401  (fake: a fixture)


def _shard(N=64, K=128, row0=0):
    return Shard4bit(packed=torch.zeros(N * K // 2, dtype=torch.uint8), absmax=torch.ones(N * K // 64),
                     absmax_8bit=None, absmax_code=None, absmax_offset=None, rows=N, row0=row0, K=K, blocksize=64,
                     quant_type="nf4")


def test_fused_routes_refuse_grad_requiring_input():
    col, row = ColumnParallelLinear4bit(_shard(), 64), RowParallelLinear4bit(_shard(), 128)
    x = torch.zeros(4, 128, requires_grad=True)
    for fn, layer in [(par.fused_forward, col), (par.fused_forward_col_sp, col), (par.fused_forward_row, row),
                      (par.fused_forward_row_sp, row)]:
        with pytest.raises(RuntimeError, match="inference only"):
            fn(layer, x, None)


@pytest.fixture
def world4(monkeypatch, fake):
    """A world of 4 seen from rank 1: the collectives record their shapes, the kernels are the fake library's."""
    calls = []

    simulate(monkeypatch, 4, 1, calls)
    monkeypatch.setattr(par, "reduce_partials", lambda parts, dtype, bias=None: parts.sum(0).to(dtype))
    monkeypatch.setattr(par, "input_grad_dequant_matmul",
                        lambda G, shard, dtype: torch.zeros(G.shape[0], shard.K, dtype=dtype))
    return calls


def test_backward_collectives_in_a_world_of_4(world4, fake):
    """Column layer: the partials all-gathered as [4, M, K] (the gradient of the gathered output read in place at this
    rank's columns), or exchanged by token under sequence parallelism; row layer: no exchange, or the token rows of
    grad_y all-gathered under sequence parallelism.  Every input gets a gradient of its shape."""
    M, K, rows = 8, 128, 64
    col = ColumnParallelLinear4bit(_shard(rows, K, row0=rows), 4 * rows)
    x = torch.zeros(M, K, dtype=torch.bfloat16, requires_grad=True)
    col._backward(torch.zeros(M, 4 * rows, dtype=torch.bfloat16), x.shape)
    sp = ColumnParallelLinear4bit(_shard(rows, K), 4 * rows, gather_output=False, sequence_parallel=True)
    assert sp._backward(torch.zeros(M, rows, dtype=torch.bfloat16), (M // 4, K)).shape == (M // 4, K)
    row = RowParallelLinear4bit(_shard(rows, K), 4 * K)
    assert row._backward(torch.zeros(M, rows, dtype=torch.bfloat16), (M, K)).shape == (M, K)
    row_sp = RowParallelLinear4bit(_shard(rows, K), 4 * K, sequence_parallel=True)
    assert row_sp._backward(torch.zeros(M // 4, rows, dtype=torch.bfloat16), (M, K)).shape == (M, K)
    assert world4 == [("all_gather_into_tensor", (4 * M * K,), (M * K,)),
                      ("all_to_all_single", (4, M // 4, K), (4, M // 4, K)),
                      ("all_gather_into_tensor", (M, rows), (M // 4, rows))]
    # every product is dequantise + cuBLAS (the fake above): no native call
    assert fake.calls == []
