"""Host side of the tensor-parallel expert layers (bitsandbytes_b200/parallel.py): the column and row cuts of a
globally quantised [E, N, K] expert tensor, the refused shapes and arguments, and, in a simulated world, the native calls
and collectives each layer's forward issues."""
import numpy as np
import pytest
import torch

import bitsandbytes_b200.backends.cuda as cb
import bitsandbytes_b200.functional as F
import bitsandbytes_b200.parallel as par
import oracle
from bitsandbytes_b200.parallel import (ColumnParallelGroupedLinear4bit, RowParallelGroupedLinear4bit,
                                        slice_grouped_weight, slice_grouped_weight_k)
from tests._parallel_sim import install_fake_lib, simulate

BF = torch.bfloat16


def _problem(E=4, N=256, K=256, bs=64, qt="nf4", nested=False, seed=5):
    """A globally quantised [E, N, K] expert tensor: (packed codes, its QuantState)."""
    g = torch.Generator().manual_seed(seed)
    W = (torch.randn(E * N, K, generator=g) / K**0.5).to(BF)
    packed, absmax = oracle.quantize_blockwise(W.float().numpy().reshape(-1), bs, qt)
    packed, absmax = torch.from_numpy(packed), torch.from_numpy(absmax)
    shape = torch.Size([E, N, K])
    if not nested:
        return packed, F.QuantState(absmax=absmax, shape=shape, code=None, blocksize=bs, quant_type=qt, dtype=BF)
    offset = absmax.mean()
    code2 = F.create_dynamic_map()
    a8, a2 = oracle.quantize_blockwise((absmax - offset).numpy(), 256, None, code2.numpy())
    s2 = F.QuantState(absmax=torch.from_numpy(a2), code=code2, blocksize=256, dtype=torch.float32)
    return packed, F.QuantState(absmax=torch.from_numpy(a8), shape=shape, code=F.get_4bit_type(qt, "cpu"), blocksize=bs,
                                quant_type=qt, dtype=BF, offset=offset, state2=s2)


def _global_scales(qs):
    if not qs.nested:
        return qs.absmax.numpy()
    return oracle.nested_absmax(qs.state2.absmax.numpy(), qs.absmax.numpy(), qs.state2.code.numpy(), float(qs.offset))


def _decode(packed, scales, bs, n, qt):
    return oracle.dequantize_blockwise(np.asarray(packed), np.asarray(scales), bs, n, qt, None, "bf16")


def _shard_decode(s):
    """A shard's [E, rows, K] weights decoded by the oracle from what the shard holds."""
    scales = s.absmax.numpy()
    if s.absmax_8bit is not None:
        scales = oracle.nested_absmax(s.absmax.numpy(), s.absmax_8bit.numpy(), s.absmax_code.numpy(),
                                      float(s.absmax_offset))
    return _decode(s.packed.numpy(), scales, s.blocksize, s.experts * s.rows * s.K, s.quant_type).reshape(
        s.experts, s.rows, s.K)


# ---------------------------------------------------------------------------------------------------- slicing
@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("bs", [32, 64, 128])
def test_column_slices_reassemble_the_global_weight(world, bs):
    """Each rank's [E, N/w, K] shard holds rows [r*N/w, (r+1)*N/w) of every expert: put side by side along N, the shards
    are the global packed codes and absmax byte for byte."""
    E, N, K = 4, 256, 256
    packed, qs = _problem(E, N, K, bs)
    shards = [slice_grouped_weight(packed, qs, world, r) for r in range(world)]
    for r, s in enumerate(shards):
        assert (s.experts, s.rows, s.row0, s.K, s.blocksize) == (E, N // world, r * N // world, K, bs)
        assert s.absmax_8bit is None and s.packed.is_contiguous() and s.absmax.is_contiguous()
    codes = torch.cat([s.packed.view(E, N // world, K // 2) for s in shards], dim=1)
    scales = torch.cat([s.absmax.view(E, N // world, K // bs) for s in shards], dim=1)
    assert torch.equal(codes.reshape(-1), packed)
    assert torch.equal(scales.reshape(-1).view(torch.int32), qs.absmax.view(torch.int32))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("bs", [32, 64, 128])
def test_row_slices_reassemble_the_global_weight(world, bs):
    """Each rank's [E, N, K/w] shard holds input features [r*K/w, (r+1)*K/w) of every expert: side by side along K, the
    global packed codes and absmax byte for byte."""
    E, N, K = 4, 128, 1024
    packed, qs = _problem(E, N, K, bs)
    shards = [slice_grouped_weight_k(packed, qs, world, r) for r in range(world)]
    for r, s in enumerate(shards):
        assert (s.experts, s.rows, s.K, s.k0) == (E, N, K // world, r * K // world)
        assert s.absmax_8bit is None
    codes = torch.cat([s.packed.view(E * N, -1) for s in shards], dim=1)
    scales = torch.cat([s.absmax.view(E * N, -1) for s in shards], dim=1)
    assert torch.equal(codes.reshape(-1), packed)
    assert torch.equal(scales.reshape(-1).view(torch.int32), qs.absmax.view(torch.int32))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("bs", [32, 64, 128])
@pytest.mark.parametrize("qt", ["nf4", "fp4"])
def test_nested_column_shards_decode_to_the_global_weights(world, bs, qt):
    """Nested statistics stay nested when every expert's slice covers whole level-2 groups of 256 blocks, and become
    plain scales otherwise; either way the shard decodes to the global weights' rows bit for bit."""
    E, N, K = 3, 256, 256
    packed, qs = _problem(E, N, K, bs, qt, nested=True)
    full = _decode(packed.numpy(), _global_scales(qs), bs, E * N * K, qt).reshape(E, N, K)
    blocks = (N // world) * K // bs
    for r in range(world):
        s = slice_grouped_weight(packed, qs, world, r)
        assert (s.absmax_8bit is not None) == (blocks % 256 == 0 and (N * K // bs) % 256 == 0)
        rows = slice(r * N // world, (r + 1) * N // world)
        assert np.array_equal(_shard_decode(s), full[:, rows])


def test_nested_column_shards_keep_and_convert():
    """Both outcomes occur: a shard of 256-block multiples keeps its nested statistics, a shard of 128 blocks does not."""
    packed, qs = _problem(4, 256, 256, 64, nested=True)
    assert slice_grouped_weight(packed, qs, 4, 1).absmax_8bit is not None   # 64 rows * 4 blocks = 256
    assert slice_grouped_weight(packed, qs, 8, 1).absmax_8bit is None       # 32 rows * 4 blocks = 128


@pytest.mark.parametrize("world", [2, 4, 8])
def test_nested_row_shards_decode_to_the_global_weights(world):
    E, N, K = 3, 64, 1024
    packed, qs = _problem(E, N, K, 64, nested=True)
    full = _decode(packed.numpy(), _global_scales(qs), 64, E * N * K, "nf4").reshape(E, N, K)
    kr = K // world
    for r in range(world):
        s = slice_grouped_weight_k(packed, qs, world, r)
        assert s.absmax_8bit is None and s.absmax.dtype == torch.float32
        assert np.array_equal(_shard_decode(s), full[:, :, r * kr:(r + 1) * kr])


def test_bad_slices_raise():
    packed, qs = _problem(4, 192, 256, 64)
    with pytest.raises(ValueError):
        slice_grouped_weight(packed, qs, 5, 0)            # 192 % 5
    with pytest.raises(ValueError):
        slice_grouped_weight(packed, qs, 2, 2)            # no rank 2
    with pytest.raises(ValueError):
        slice_grouped_weight_k(packed, qs, 8, 0)          # 256 % (8 * 64)
    with pytest.raises(ValueError):
        slice_grouped_weight_k(packed, qs, 3, 0)
    flat = F.QuantState(absmax=qs.absmax, shape=torch.Size([4 * 192, 256]), blocksize=64, quant_type="nf4", dtype=BF)
    with pytest.raises(ValueError):
        slice_grouped_weight(packed, flat, 2, 0)          # not an [E, N, K] state
    with pytest.raises(ValueError):
        slice_grouped_weight_k(packed, flat, 2, 0)
    packed, qs = _problem(2, 64, 32 * 3, 64)              # K % blocksize
    with pytest.raises(ValueError):
        slice_grouped_weight(packed, qs, 2, 0)


# ---------------------------------------------------------------------------------------------------- wrappers
def _grouped_args(M=8, E=4, N=64, K=128, bs=64, dtype=BF):
    A = torch.zeros(M, K, dtype=dtype)
    B = torch.zeros(E * N * K // 2, dtype=torch.uint8)
    absmax = torch.ones(E * N * K // bs)
    offs = torch.zeros(E, dtype=torch.int32)
    return A, B, (E, N, K), absmax, bs, offs


def test_wrappers_refuse_bad_arguments_before_any_launch(monkeypatch):
    lib = install_fake_lib(monkeypatch)
    A, B, shape, absmax, bs, offs = _grouped_args()
    M, (E, N, K) = A.shape[0], shape
    part = torch.empty(M, N)
    out = torch.empty(M, N, dtype=BF)
    wide = torch.empty(M, N + 8, dtype=BF)

    def partial(o=part, ldc=N, **kw):
        args = dict(A=A, B=B, shapeB=shape, absmax=absmax, blocksize=bs, quant_type="nf4", offs=offs)
        args.update(kw)
        return cb.gemm_4bit_grouped_partial(**args, out=o, ldc=ldc)

    def into(o=out, ldc=N, bias=None):
        return cb.gemm_4bit_grouped_into(A, B, shape, absmax, bs, "nf4", offs, bias, None, None, None, o, ldc)

    bad = [
        (lambda: partial(ldc=N - 1), "row stride"),                                 # ldc < N
        (lambda: partial(torch.empty(M - 1, N)), r"out must be \[8, 64\]"),       # too few rows
        (lambda: partial(out), "destinations must be torch.float32"),               # not fp32
        (lambda: partial(torch.empty(N, M).t()), "unit column stride"),             # transposed
        (lambda: partial(torch.empty(M, 2 * N)[:, ::2]), "unit column stride"),     # column-strided
        (lambda: partial(torch.empty(M, N + 8)[:, :N], ldc=N), "row stride"),       # ldc is not the row stride
        (lambda: partial(mt=256), "mt must be"),                                    # tile
        (lambda: partial(absmax=absmax[1:]), "absmax must hold"),                   # scales
        (lambda: partial(A=A.float()), "float16 or bfloat16"),                      # fp32 A
        (lambda: partial(offs=offs[1:]), "offs must be int32"),                     # offs [E]
        (lambda: into(ldc=N - 1), "row stride"),
        (lambda: into(part), "destinations must be torch.bfloat16"),
        (lambda: into(torch.empty(N, M, dtype=BF).t()), "unit column stride"),
        (lambda: into(wide[:, :N], N), "row stride"),
        (lambda: into(bias=torch.zeros(N, dtype=BF)), "bias must be"),              # bias [E, N]
    ]
    for call, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            call()
    assert lib.calls == []
    into(wide[:, :N], N + 8)  # a column slice of a wider buffer at its row stride is served
    assert [n for n, _ in lib.calls] == ["cbnb_b200_gemm_4bit_grouped"]


def test_grouped_reduce_refuses_bad_arguments_before_any_launch(monkeypatch):
    """Every check of the reduction runs before its device check, so host tensors reach each of them."""
    lib = install_fake_lib(monkeypatch)
    E, M, N = 4, 8, 64
    parts = torch.zeros(2, M, N)
    offs = torch.zeros(E, dtype=torch.int32)
    bad = [
        (dict(parts=parts.to(torch.float16)), "parts must be"),
        (dict(parts=parts[0]), "parts must be"),
        (dict(dtype=torch.float32), "dtype must be"),
        (dict(parts=torch.zeros(0, M, N)), "no partials"),
        (dict(offs=offs.long()), "offs must be int32"),
        (dict(offs=offs.view(2, 2)), "offs must be int32"),
        (dict(offs=torch.zeros(0, dtype=torch.int32)), "offs must be int32"),
        (dict(offs=torch.zeros(1025, dtype=torch.int32)), "offs must be int32"),
        (dict(bias=torch.zeros(E, N, dtype=torch.float16)), "bias must be"),
        (dict(bias=torch.zeros(N, dtype=BF)), "bias must be"),
        (dict(bias=torch.zeros(E + 1, N, dtype=BF)), "bias must be"),
        (dict(out=torch.empty(M, N, dtype=torch.float16)), "out must be"),
        (dict(out=torch.empty(M + 1, N, dtype=BF)), "out must be"),
        (dict(out=torch.empty(N, M, dtype=BF).t()), "out must be"),
        ({}, "CUDA device"),  # every argument right: refused only for being on the host
    ]
    for kw, msg in bad:
        args = dict(parts=parts, offs=offs, dtype=BF, bias=torch.zeros(E, N, dtype=BF), out=None)
        args.update(kw)
        with pytest.raises(RuntimeError, match=msg):
            cb.reduce_partials_grouped(args["parts"], args["offs"], args["dtype"], args["bias"], args["out"])
    assert lib.calls == []


# ---------------------------------------------------------------------------------------------------- simulated world
class World:
    """Rank ``rank`` of a simulated world of ``world``: ``log`` holds every native call (name, scalars, destinations),
    collective and reduction, in order."""

    def __init__(self, monkeypatch, world, rank):
        self.log = []
        self.lib = install_fake_lib(monkeypatch, self.log)
        simulate(monkeypatch, world, rank, self.log)
        log = self.log

        def reduce_grouped(parts, offs, dtype, bias=None, out=None):
            log.append(("reduce_partials_grouped", tuple(parts.shape), tuple(offs.shape), dtype,
                        None if bias is None else tuple(bias.shape)))
            return torch.zeros(parts.shape[1:], dtype=dtype)

        monkeypatch.setattr(par, "reduce_partials_grouped", reduce_grouped)


E, N, K, M = 4, 256, 512, 24
QT_NF4, BF_ID = 2, 2


def _column_layer(world, rank, bias=True, gather_output=True):
    packed, qs = _problem(E, N, K, 64)
    b = torch.randn(E, N).to(BF) if bias else None
    return ColumnParallelGroupedLinear4bit(slice_grouped_weight(packed, qs, world, rank), N, b,
                                           gather_output=gather_output), b


@pytest.mark.parametrize("world,rank", [(1, 0), (4, 1), (8, 7)])
@pytest.mark.parametrize("gather", [True, False])
def test_column_layer_calls(monkeypatch, world, rank, gather):
    w = World(monkeypatch, world, rank)
    layer, b = _column_layer(world, rank, gather_output=gather)
    rows = N // world
    assert torch.equal(layer.bias_shard, b[:, rank * rows:(rank + 1) * rows])
    x = torch.zeros(M, K, dtype=BF)
    offs = torch.tensor([5, 5, 17, 20], dtype=torch.int32)
    y = layer(x, offs)
    gathered = gather and world > 1
    assert y.shape == (M, N if gathered else rows)
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, offs, E, out, bias, M, N, K, ldc, bs, qt, dtype, stream)
    want = [("gemm_4bit_grouped", (E, M, rows, K, rows, 64, QT_NF4, BF_ID, 0), None)]
    if gathered:
        want.append(("all_gather_into_tensor", (world * M * rows,), (M * rows,)))
        (_, args), = w.lib.calls
        assert args[8] == layer._stage[rank].data_ptr()  # this rank's slot of the stage
    assert w.log == want


@pytest.mark.parametrize("world,rank", [(1, 0), (2, 1), (8, 3)])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("input_is_parallel", [True, False])
def test_row_layer_calls(monkeypatch, world, rank, bias, input_is_parallel):
    w = World(monkeypatch, world, rank)
    Kd, Nd = 1024, 128  # down: in_features = the intermediate size, out_features = hidden
    packed, qs = _problem(E, Nd, Kd, 64)
    b = torch.randn(E, Nd).to(BF) if bias else None
    layer = RowParallelGroupedLinear4bit.from_quantized(packed, qs, b, input_is_parallel=input_is_parallel)
    kr = Kd // world
    assert (layer.shard.experts, layer.shard.rows, layer.shard.K, layer.shard.k0) == (E, Nd, kr, rank * kr)
    x = torch.zeros(M, kr if input_is_parallel else Kd, dtype=BF)
    offs = torch.tensor([3, 9, 9, 24], dtype=torch.int32)
    y = layer(x, offs)
    assert y.shape == (M, Nd)
    # (A, B, absmax, offs, E, out, M, N, K, ldc, bs, qt, dtype, mt, stream)
    want = [("gemm_4bit_grouped_partial", (E, M, Nd, kr, Nd, 64, QT_NF4, BF_ID, 0, 0), None)]
    if world > 1:
        want.append(("all_gather_into_tensor", (world * M * Nd,), (M * Nd,)))
    want.append(("reduce_partials_grouped", (world, M, Nd), (E,), BF, (E, Nd) if bias else None))
    assert w.log == want
    (_, args), = w.lib.calls
    assert args[5] == layer._stage[rank].data_ptr()


def test_layers_refuse_training_sequence_parallel_and_fused_routes(monkeypatch):
    World(monkeypatch, 2, 0)
    col, _ = _column_layer(2, 0)
    packed, qs = _problem(E, 128, 1024, 64)
    row = RowParallelGroupedLinear4bit.from_quantized(packed, qs)
    offs = torch.tensor([3, 9, 9, 24], dtype=torch.int32)
    for layer, width in ((col, K), (row, 512)):
        x = torch.zeros(M, width, dtype=BF, requires_grad=True)
        with pytest.raises(RuntimeError, match="inference only"):
            layer(x, offs)
        with torch.no_grad():
            layer(x, offs)  # the same input without grad runs
    with pytest.raises(ValueError, match="sequence_parallel"):
        ColumnParallelGroupedLinear4bit(col.shard, N, gather_output=False, sequence_parallel=True)
    with pytest.raises(ValueError, match="sequence_parallel"):
        RowParallelGroupedLinear4bit.from_quantized(packed, qs, sequence_parallel=True)
    with pytest.raises(RuntimeError, match="symmetric-memory"):
        par.fused_forward(col, torch.zeros(M, K, dtype=BF), peers=None)
    with pytest.raises(RuntimeError, match="symmetric-memory"):
        par.fused_forward_row(row, torch.zeros(M, 512, dtype=BF), peers=None)
