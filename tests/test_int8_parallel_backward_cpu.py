"""CPU tests of the tensor-parallel LLM.int8() backward: the argument checks of the one-pass weight dequantisation
(against a fake library), the refusal of grad-requiring input by the symmetric-memory routes, and the collectives the
backward runs in a simulated world of 4."""
import pytest
import torch

import bitsandbytes_b200.backends.cuda as cb
import bitsandbytes_b200.parallel as par
from bitsandbytes_b200.parallel import ColumnParallelLinear8bitLt, RowParallelLinear8bitLt, Shard8bit
from tests._parallel_sim import fake, simulate  # noqa: F401  (fake: a fixture)


def test_dequant_rows_wrapper_checks(fake):
    """Bad codes, scales, dtypes or outputs raise RuntimeError before any native call; a good call passes the row
    stride of its output, the shape and the dtype."""
    CB, SCB = torch.zeros(6, 40, dtype=torch.int8), torch.ones(6)
    bf16 = torch.bfloat16

    def call(CB=CB, SCB=SCB, dtype=bf16, out=None):
        return cb.int8_dequant_rows(CB, SCB, dtype, out)

    bad = [dict(CB=CB.float()),                                                   # not int8
           dict(CB=torch.zeros(240, dtype=torch.int8)),                           # not 2-D
           dict(SCB=torch.ones(5)),                                               # one scale per row
           dict(SCB=torch.ones(6, dtype=torch.float16)),                          # fp32 scales
           dict(dtype=torch.float32),                                             # fp16 / bf16 only
           dict(dtype=torch.int8),
           dict(out=torch.zeros(6, 40)),                                          # out of another dtype
           dict(out=torch.zeros(6, 39, dtype=bf16)),                              # out shape
           dict(out=torch.zeros(40, 6, dtype=bf16).t()),                          # column stride
           dict(out=torch.zeros(240, dtype=bf16).as_strided((6, 40), (39, 1)))]   # ldo < cols
    for kw in bad:
        with pytest.raises(RuntimeError, match="int8_dequant_rows"):
            call(**kw)
    assert fake.calls == []
    out = call()
    assert out.shape == (6, 40) and out.dtype == bf16
    wide = torch.zeros(6, 48, dtype=torch.float16)
    assert call(dtype=torch.float16, out=wide[:, :40]).data_ptr() == wide.data_ptr()
    assert call(CB=torch.zeros(0, 40, dtype=torch.int8), SCB=torch.ones(0)).shape == (0, 40)
    assert [n for n, _ in fake.calls] == ["cbnb_b200_int8_dequant_rows"] * 2
    # (CB, SCB, out, ldo, rows, cols, dtype, stream)
    assert [a[3:7] for _, a in fake.calls] == [(40, 6, 40, 2), (48, 6, 40, 1)]


def _shard(rows=64, K=128, row0=0, k0=0):
    return Shard8bit(CB=torch.zeros(rows, K, dtype=torch.int8), SCB=torch.ones(rows), rows=rows, row0=row0, K=K, k0=k0)


def test_fused_routes_refuse_grad_requiring_input():
    col = ColumnParallelLinear8bitLt(_shard(), 64)
    row = RowParallelLinear8bitLt(_shard(), 128)
    x = torch.zeros(4, 128, dtype=torch.float16, requires_grad=True)
    for fn, layer in [(par.fused_forward_col8, col), (par.fused_forward_col8_sp, col), (par.fused_forward_row8, row),
                      (par.fused_forward_row8_sp, row)]:
        with pytest.raises(RuntimeError, match="inference only"):
            fn(layer, x, None)


@pytest.fixture
def world4(monkeypatch, fake):
    """A world of 4 seen from rank 1: the collectives record their shapes, the weight is the torch expression of
    MatMul8bitLt.backward and the products run on the CPU."""
    calls = []

    def dequant_rows(CB, SCB, dtype):
        calls.append(("int8_dequant_rows", tuple(CB.shape), dtype))
        return CB.to(dtype, copy=True).mul_(SCB.unsqueeze(1).mul(1.0 / 127.0))

    simulate(monkeypatch, 4, 1, calls)
    monkeypatch.setattr(par, "reduce_partials", lambda parts, dtype, bias=None: parts.sum(0).to(dtype))
    monkeypatch.setattr(par, "int8_dequant_rows", dequant_rows)
    monkeypatch.setattr(par, "input_grad_dequant_matmul",
                        lambda G, shard, dtype: (G.float() @ shard.dequantize(G.dtype).float()).to(dtype))
    return calls


def test_backward_collectives_in_a_world_of_4(world4, fake):
    """Every row of the backward's table: the column layer's fp32 partials all-gathered as [4, M, K] (the gathered
    output's gradient read at this rank's columns, or the local output's gradient), or exchanged by token under
    sequence parallelism; the row layer with no exchange, the token rows of grad_y all-gathered under sequence
    parallelism, or the ranks' input columns all-gathered for the whole input.  Every input gets a gradient of its
    shape, every product a weight of the gradient's dtype, and no native call is made besides."""
    M, K, rows = 8, 128, 64
    bf16 = torch.bfloat16
    g = torch.Generator().manual_seed(0)
    CB = torch.randint(-128, 128, (rows, K), generator=g, dtype=torch.int8)
    SCB = torch.rand(rows, generator=g) + 0.5
    shard = Shard8bit(CB=CB, SCB=SCB, rows=rows, row0=rows, K=K)
    W = CB.float() * SCB.unsqueeze(1).mul(1.0 / 127.0)
    gy = torch.randn(M, 4 * rows, generator=g).to(bf16)
    col = ColumnParallelLinear8bitLt(shard, 4 * rows)
    got = col._backward(gy, (M, K))
    # the simulated gather repeats this rank's partial G_1 . W_1 (its columns of the gathered gradient)
    P = gy[:, rows:2 * rows].float() @ W.to(bf16).float()
    want = torch.stack([P] * 4).sum(0).to(bf16)
    assert got.shape == (M, K) and torch.equal(got, want)
    local = ColumnParallelLinear8bitLt(shard, 4 * rows, gather_output=False)
    assert local._backward(gy[:, rows:2 * rows], (M, K)).shape == (M, K)
    sp = ColumnParallelLinear8bitLt(shard, 4 * rows, gather_output=False, sequence_parallel=True)
    assert sp._backward(gy[:, :rows].reshape(2, M // 2, rows), (M // 4, K)).shape == (M // 4, K)

    kshard = Shard8bit(CB=CB.t().contiguous(), SCB=torch.ones(K), rows=K, row0=0, K=rows, k0=rows)
    row = RowParallelLinear8bitLt(kshard, 4 * rows)
    assert row._backward(torch.zeros(M, K, dtype=bf16), (M, rows)).shape == (M, rows)
    row_sp = RowParallelLinear8bitLt(kshard, 4 * rows, sequence_parallel=True)
    assert row_sp._backward(torch.zeros(M // 4, K, dtype=bf16), (M, rows)).shape == (M, rows)
    whole = RowParallelLinear8bitLt(kshard, 4 * rows, input_is_parallel=False)
    assert whole._backward(torch.zeros(2, M // 2, K, dtype=bf16), (2, M // 2, 4 * rows)).shape == (2, M // 2, 4 * rows)
    dq_col, dq_row = ("int8_dequant_rows", (rows, K), bf16), ("int8_dequant_rows", (K, rows), bf16)
    assert world4 == [dq_col, ("all_gather_into_tensor", (4 * M * K,), (M * K,)),
                      dq_col, ("all_gather_into_tensor", (4 * M * K,), (M * K,)),
                      dq_col, ("all_to_all_single", (4, M // 4, K), (4, M // 4, K)),
                      dq_row,
                      ("all_gather_into_tensor", (M, K), (M // 4, K)), dq_row,
                      dq_row, ("all_gather_into_tensor", (4, M, rows), (M, rows))]
    assert fake.calls == []
