"""CPU tests of the forward protocol of the tensor-parallel layers and their symmetric-memory routes
(``fused_forward*``): in a simulated world of 4 seen from rank 1, and in a world of 1, the ordered list of native calls
(with their scalar arguments and destination lists), NCCL collectives, symmetric-memory slots taken, peer copies,
barriers and reductions that each forward issues.  The statistics the fake library cannot produce (outlier columns, the
reductions) come from recording stand-ins."""
import pytest
import torch

import bitsandbytes_b200.functional as F
import bitsandbytes_b200.parallel as par
from bitsandbytes_b200.parallel import (ColumnParallelLinear4bit, ColumnParallelLinear8bitLt, RowParallelLinear4bit,
                                        RowParallelLinear8bitLt, Shard4bit, Shard8bit)
from tests._parallel_sim import install_fake_lib, peer_ptrs, simulate

M, K, N = 8, 128, 256   # tokens, in_features, out_features of the column layers (the row layers: N -> K)
BF = torch.bfloat16


class World:
    """One rank of a simulated world: ``log`` holds every event in order, ``lib`` is the fake native library."""

    def __init__(self, monkeypatch, world, rank, outliers=0):
        self.world, self.rank, self.log = world, rank, []
        self.lib = install_fake_lib(monkeypatch, self.log)
        simulate(monkeypatch, world, rank, self.log)
        log = self.log
        slot = par._PeerSlots.slot

        def take(peers):
            got = slot(peers)
            log.append(("slot", got[2].slot))
            return got

        def cols(width):  # the first ``outliers`` input features of this rank hold an outlier
            flags = torch.zeros(width, dtype=torch.int32)
            flags[:outliers] = 1
            return flags

        def vectorwise_quant(A, threshold=0.0):
            log.append(("int8_vectorwise_quant", tuple(A.shape), threshold))
            c = torch.nonzero(cols(A.shape[1])).view(-1) if threshold > 0.0 else None
            return torch.zeros(A.shape, dtype=torch.int8), torch.ones(A.shape[0]), c

        def quant_flags(A, threshold):
            log.append(("int8_vectorwise_quant_flags", tuple(A.shape), threshold))
            return (torch.zeros(A.shape, dtype=torch.int8), torch.ones(A.shape[0]),
                    cols(A.shape[1]) if threshold > 0.0 else None)

        def row_stats(A, threshold):
            log.append(("int8_row_stats", tuple(A.shape), threshold))
            return torch.ones(A.shape[0]), cols(A.shape[1]) if threshold > 0.0 else None

        def quant_with_stats(A, SCA, threshold):
            log.append(("int8_quant_with_stats", tuple(A.shape), tuple(SCA.shape), threshold))
            return torch.zeros(A.shape, dtype=torch.int8)

        def reduce_partials(parts, dtype, bias=None):
            log.append(("reduce_partials", tuple(parts.shape), dtype, bias is not None))
            return torch.zeros(parts.shape[1:], dtype=dtype)

        def int8_reduce(parts, SCA, SCB, dtype, bias=None, subA=None, subBT=None, out=None):
            log.append(("int8_reduce_partials", tuple(parts.shape), tuple(SCA.shape), dtype,
                        None if subA is None else tuple(subA.shape), None if subBT is None else tuple(subBT.shape)))
            return torch.zeros(parts.shape[1:], dtype=dtype)

        monkeypatch.setattr(par._PeerSlots, "slot", take)
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
        monkeypatch.setattr(F, "int8_vectorwise_quant", vectorwise_quant)
        monkeypatch.setattr(par, "int8_vectorwise_quant_flags", quant_flags)
        monkeypatch.setattr(par, "int8_row_stats", row_stats)
        monkeypatch.setattr(par, "int8_quant_with_stats", quant_with_stats)
        monkeypatch.setattr(par, "reduce_partials", reduce_partials)
        monkeypatch.setattr(par, "int8_reduce_partials", int8_reduce)

    def ptrs(self, slot, offset, own_first=True):
        """The destinations of a slot ``offset`` bytes into every rank's buffer: this rank's first, or in rank order."""
        bases = peer_ptrs(slot, self.world)
        order = ([self.rank] + [r for r in range(self.world) if r != self.rank]) if own_first else range(self.world)
        return [bases[r] + offset for r in order]


def _col4(w, sp=False, gather=True):
    rows = N // w.world
    shard = Shard4bit(packed=torch.zeros(rows * K // 2, dtype=torch.uint8), absmax=torch.ones(rows * K // 64),
                      absmax_8bit=None, absmax_code=None, absmax_offset=None, rows=rows, row0=w.rank * rows, K=K,
                      blocksize=64, quant_type="nf4")
    return ColumnParallelLinear4bit(shard, N, torch.zeros(N, dtype=BF), gather_output=gather and not sp,
                                    sequence_parallel=sp)


def _row4(w, sp=False, input_is_parallel=True):
    kr = N // w.world
    shard = Shard4bit(packed=torch.zeros(K * kr // 2, dtype=torch.uint8), absmax=torch.ones(K * kr // 64),
                      absmax_8bit=None, absmax_code=None, absmax_offset=None, rows=K, row0=0, K=kr, blocksize=64,
                      quant_type="nf4", k0=w.rank * kr)
    return RowParallelLinear4bit(shard, N, torch.zeros(K, dtype=BF), input_is_parallel=input_is_parallel,
                                 sequence_parallel=sp)


def _col8(w, threshold, sp=False, gather=True):
    rows = N // w.world
    shard = Shard8bit(CB=torch.zeros(rows, K, dtype=torch.int8), SCB=torch.ones(rows), rows=rows, row0=w.rank * rows,
                      K=K)
    return ColumnParallelLinear8bitLt(shard, N, torch.zeros(N, dtype=BF), gather_output=gather and not sp,
                                      threshold=threshold, sequence_parallel=sp)


def _row8(w, threshold, sp=False):
    kr = N // w.world
    shard = Shard8bit(CB=torch.zeros(K, kr, dtype=torch.int8), SCB=torch.ones(K), rows=K, row0=0, K=kr,
                      k0=w.rank * kr)
    return RowParallelLinear8bitLt(shard, N, torch.zeros(K, dtype=BF), threshold=threshold, sequence_parallel=sp)


def _x(*shape):
    return torch.zeros(shape, dtype=BF)


def _gather(w):
    return par.PeerGather(M, N, BF, "cpu")


def _parts(w, dtype=torch.float32):
    return par.PeerPartials(M, K, "cpu", dtype=dtype)


def _parts_sp(w, dtype=torch.float32):
    return par.PeerPartials(M // w.world, K, "cpu", dtype=dtype)


# id -> (world, outlier columns per rank, refused native calls, the forward); the events each issues are in EVENTS
_GEMM4, _PARTIAL, _SCATTER4 = "cbnb_b200_gemm_4bit_multi_out", "cbnb_b200_gemm_4bit_partial", \
    "cbnb_b200_gemm_4bit_partial_scatter"
_GEMM8, _SCATTER8 = "cbnb_b200_int8_gemm_multi_out", "cbnb_b200_int8_gemm_partial_scatter"
CASES = {}
for _w in (4, 1):
    _n = N // _w
    CASES.update({
        f"col4-w{_w}": (_w, 0, (), lambda w: _col4(w)(_x(M, K))),
        f"fused_forward-w{_w}": (_w, 0, (), lambda w: par.fused_forward(_col4(w), _x(M, K), _gather(w))),
        f"fused_forward-refused-w{_w}": (_w, 0, (_GEMM4,),
                                         lambda w: par.fused_forward(_col4(w), _x(M, K), _gather(w))),
        f"row4-w{_w}": (_w, 0, (), lambda w, n=_n: _row4(w)(_x(M, n))),
        f"fused_forward_row-w{_w}": (_w, 0, (), lambda w, n=_n: par.fused_forward_row(_row4(w), _x(M, n), _parts(w))),
        f"fused_forward_row-refused-w{_w}": (_w, 0, (_PARTIAL,),
                                             lambda w, n=_n: par.fused_forward_row(_row4(w), _x(M, n), _parts(w))),
        f"row8-refused-w{_w}": (_w, 0, (_GEMM8,), lambda w, n=_n: _row8(w, 0.0)(_x(M, n))),
        f"fused_forward_row8-refused-w{_w}": (_w, 0, (_GEMM8,), lambda w, n=_n: par.fused_forward_row8(
            _row8(w, 0.0), _x(M, n), _parts(w, torch.int32))),
    })
    # int8: threshold 0, a few outlier columns (the GEMM epilogue's), more than 64 in all (the addmm chain)
    for _thr, _J, _tag in ((0.0, 0, "t0"), (6.0, 2, "j2"), (6.0, 65 if _w == 1 else 17, "j65")):
        _Jc = 65 if _tag == "j65" else _J  # the column layers see all K features, the row layers K / world
        CASES.update({
            f"col8-{_tag}-w{_w}": (_w, _Jc, (), lambda w, t=_thr: _col8(w, t)(_x(M, K))),
            f"fused_forward_col8-{_tag}-w{_w}": (_w, _Jc, (), lambda w, t=_thr: par.fused_forward_col8(
                _col8(w, t), _x(M, K), _gather(w))),
            f"row8-{_tag}-w{_w}": (_w, _J, (), lambda w, t=_thr, n=_n: _row8(w, t)(_x(M, n))),
            f"fused_forward_row8-{_tag}-w{_w}": (_w, _J, (), lambda w, t=_thr, n=_n: par.fused_forward_row8(
                _row8(w, t), _x(M, n), _parts(w, torch.int32))),
        })
_n = N // 4
CASES.update({
    "col4-sp": (4, 0, (), lambda w: _col4(w, sp=True)(_x(M // 4, K))),
    "fused_forward_col_sp": (4, 0, (), lambda w: par.fused_forward_col_sp(_col4(w, sp=True), _x(M // 4, K),
                                                                          par.PeerGather(M, K, BF, "cpu"))),
    "row4-sp": (4, 0, (), lambda w: _row4(w, sp=True)(_x(M, _n))),
    "fused_forward_row_sp": (4, 0, (), lambda w: par.fused_forward_row_sp(_row4(w, sp=True), _x(M, _n), _parts_sp(w))),
    "fused_forward_row_sp-refused": (4, 0, (_SCATTER4,), lambda w: par.fused_forward_row_sp(
        _row4(w, sp=True), _x(M, _n), _parts_sp(w))),
    "fused_forward_row8_sp-refused": (4, 0, (_SCATTER8,), lambda w: par.fused_forward_row8_sp(
        _row8(w, 0.0, sp=True), _x(M, _n), _parts_sp(w, torch.int32))),
})
for _thr, _J, _tag in ((0.0, 0, "t0"), (6.0, 2, "j2"), (6.0, 17, "j65")):
    _Jc = 65 if _tag == "j65" else _J
    CASES.update({
        f"col8-sp-{_tag}": (4, _Jc, (), lambda w, t=_thr: _col8(w, t, sp=True)(_x(M // 4, K))),
        f"fused_forward_col8_sp-{_tag}": (4, _Jc, (), lambda w, t=_thr: par.fused_forward_col8_sp(
            _col8(w, t, sp=True), _x(M // 4, K), par.PeerInt8Input(M, K, "cpu"))),
        f"row8-sp-{_tag}": (4, _J, (), lambda w, t=_thr: _row8(w, t, sp=True)(_x(M, _n))),
        f"fused_forward_row8_sp-{_tag}": (4, _J, (), lambda w, t=_thr: par.fused_forward_row8_sp(
            _row8(w, t, sp=True), _x(M, _n), _parts_sp(w, torch.int32))),
    })


def _run(monkeypatch, case):
    world, outliers, refuse, fn = CASES[case]
    w = World(monkeypatch, world, 1 if world > 1 else 0, outliers)
    w.lib.refuse |= set(refuse)
    try:
        result = tuple(fn(w).shape)
    except RuntimeError as e:
        result = str(e)
    return result, w.log


F32, I32, I8 = torch.float32, torch.int32, torch.int8
# (output shape or the RuntimeError's message, the events in order); a native call is (name, its scalar arguments, its
# destinations: a symmetric-memory address, or "t" for a tensor)
EVENTS = {
    'col4-w4': ((8, 256), [
        ('gemm_4bit_strided', (8, 64, 128, 64, 64, 2, 2, 0), None),
        ('all_gather_into_tensor', (2048,), (512,)),
    ]),
    'fused_forward-w4': ((8, 256), [
        ('slot', 0),
        ('gemm_4bit_multi_out', (4, 8, 64, 128, 256, 64, 2, 2, 0), [1010128, 1000128, 1020128, 1030128]),
        ('barrier', 0),
    ]),
    'fused_forward-refused-w4': ((8, 256), [
        ('slot', 0),
        ('gemm_4bit_multi_out', (4, 8, 64, 128, 256, 64, 2, 2, 0), [1010128, 1000128, 1020128, 1030128]),
        ('gemm_4bit_strided', (8, 64, 128, 64, 64, 2, 2, 0), None),
        ('all_gather_into_tensor', (2048,), (512,)),
        ('barrier', 0),
    ]),
    'row4-w4': ((8, 128), [
        ('gemm_4bit_partial', (1, 8, 128, 64, 128, 64, 2, 2, 0), ['t']),
        ('all_gather_into_tensor', (4096,), (1024,)),
        ('reduce_partials', (4, 8, 128), BF, True),
    ]),
    'fused_forward_row-w4': ((8, 128), [
        ('slot', 0),
        ('gemm_4bit_partial', (4, 8, 128, 64, 128, 64, 2, 2, 0), [1014096, 1004096, 1024096, 1034096]),
        ('barrier', 0),
        ('reduce_partials', (4, 8, 128), BF, True),
    ]),
    'fused_forward_row-refused-w4': ('gemm_4bit_partial does not serve this shard shape', [
        ('slot', 0),
        ('gemm_4bit_partial', (4, 8, 128, 64, 128, 64, 2, 2, 0), [1014096, 1004096, 1024096, 1034096]),
    ]),
    'row8-refused-w4': ('the int8 GEMM does not serve this shard shape', [
        ('int8_row_stats', (8, 64), 0.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 0.0),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 64, 128, 0, 0), ['t']),
    ]),
    'fused_forward_row8-refused-w4': ('the int8 GEMM does not serve this shard shape', [
        ('int8_row_stats', (8, 64), 0.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 0.0),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 4, 8, 128, 64, 128, 0, 0), [1014096, 1004096, 1024096, 1034096]),
    ]),
    'col8-t0-w4': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 0.0),
        ('int8_gemm_multi_out', (0, 1, 8, 64, 128, 64, 2, 0), ['t']),
        ('all_gather_into_tensor', (2048,), (512,)),
    ]),
    'fused_forward_col8-t0-w4': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 0.0),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 4, 8, 64, 128, 256, 2, 0), [1010128, 1000128, 1020128, 1030128]),
        ('barrier', 0),
    ]),
    'row8-t0-w4': ((8, 128), [
        ('int8_row_stats', (8, 64), 0.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 0.0),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 64, 128, 0, 0), ['t']),
        ('all_gather_into_tensor', (4096,), (1024,)),
        ('int8_reduce_partials', (4, 8, 128), (8,), BF, None, None),
    ]),
    'fused_forward_row8-t0-w4': ((8, 128), [
        ('int8_row_stats', (8, 64), 0.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 0.0),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 4, 8, 128, 64, 128, 0, 0), [1014096, 1004096, 1024096, 1034096]),
        ('barrier', 0),
        ('int8_reduce_partials', (4, 8, 128), (8,), BF, None, None),
    ]),
    'col8-j2-w4': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 6.0),
        ('int8_outlier_prep', (2, 8, 8, 64, 128, 2, 0), None),
        ('int8_gemm_multi_out', (8, 1, 8, 64, 128, 64, 2, 0), ['t']),
        ('all_gather_into_tensor', (2048,), (512,)),
    ]),
    'fused_forward_col8-j2-w4': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 6.0),
        ('slot', 0),
        ('int8_outlier_prep', (2, 8, 8, 64, 128, 2, 0), None),
        ('int8_gemm_multi_out', (8, 4, 8, 64, 128, 256, 2, 0), [1010128, 1000128, 1020128, 1030128]),
        ('barrier', 0),
    ]),
    'row8-j2-w4': ((8, 128), [
        ('int8_row_stats', (8, 64), 6.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 6.0),
        ('int8_zero_columns', (2, 8, 64, 0), None),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 64, 128, 0, 0), ['t']),
        ('all_gather_into_tensor', (4096,), (1024,)),
        ('all_gather_into_tensor', (4,), (1,)),
        ('int8_outlier_prep', (2, 8, 8, 128, 64, 2, 0), None),
        ('all_gather_into_tensor', (4352,), (1088,)),
        ('int8_reduce_partials', (4, 8, 128), (8,), BF, (8, 8), (128, 8)),
    ]),
    'fused_forward_row8-j2-w4': ((8, 128), [
        ('int8_row_stats', (8, 64), 6.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 6.0),
        ('int8_zero_columns', (2, 8, 64, 0), None),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 4, 8, 128, 64, 128, 0, 0), [1014096, 1004096, 1024096, 1034096]),
        ('all_gather_into_tensor', (4,), (1,)),
        ('int8_outlier_prep', (2, 8, 8, 128, 64, 2, 0), None),
        ('all_gather_into_tensor', (4352,), (1088,)),
        ('barrier', 0),
        ('int8_reduce_partials', (4, 8, 128), (8,), BF, (8, 8), (128, 8)),
    ]),
    'col8-j65-w4': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 6.0),
        ('int8_gemm_multi_out', (0, 1, 8, 64, 128, 64, 2, 0), ['t']),
        ('all_gather_into_tensor', (2048,), (512,)),
        ('all_gather_into_tensor', (256, 65), (64, 65)),
    ]),
    'fused_forward_col8-j65-w4': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 6.0),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 1, 8, 64, 128, 64, 2, 0), ['t']),
        ('all_gather_into_tensor', (2048,), (512,)),
        ('all_gather_into_tensor', (256, 65), (64, 65)),
        ('barrier', 0),
    ]),
    'row8-j65-w4': ((8, 128), [
        ('int8_row_stats', (8, 64), 6.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 6.0),
        ('int8_zero_columns', (17, 8, 64, 0), None),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 64, 128, 0, 0), ['t']),
        ('all_gather_into_tensor', (4096,), (1024,)),
        ('all_gather_into_tensor', (4,), (1,)),
        ('int8_outlier_prep', (17, 24, 8, 128, 64, 2, 0), None),
        ('all_gather_into_tensor', (13056,), (3264,)),
        ('int8_reduce_partials', (4, 8, 128), (8,), BF, None, None),
    ]),
    'fused_forward_row8-j65-w4': ((8, 128), [
        ('int8_row_stats', (8, 64), 6.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 6.0),
        ('int8_zero_columns', (17, 8, 64, 0), None),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 4, 8, 128, 64, 128, 0, 0), [1014096, 1004096, 1024096, 1034096]),
        ('all_gather_into_tensor', (4,), (1,)),
        ('int8_outlier_prep', (17, 24, 8, 128, 64, 2, 0), None),
        ('all_gather_into_tensor', (13056,), (3264,)),
        ('barrier', 0),
        ('int8_reduce_partials', (4, 8, 128), (8,), BF, None, None),
    ]),
    'col4-w1': ((8, 256), [
        ('gemm_4bit_strided', (8, 256, 128, 256, 64, 2, 2, 0), None),
    ]),
    'fused_forward-w1': ((8, 256), [
        ('slot', 0),
        ('gemm_4bit_multi_out', (1, 8, 256, 128, 256, 64, 2, 2, 0), [1000000]),
        ('barrier', 0),
    ]),
    'fused_forward-refused-w1': ((8, 256), [
        ('slot', 0),
        ('gemm_4bit_multi_out', (1, 8, 256, 128, 256, 64, 2, 2, 0), [1000000]),
        ('gemm_4bit_strided', (8, 256, 128, 256, 64, 2, 2, 0), None),
        ('all_gather_into_tensor', (2048,), (2048,)),
        ('barrier', 0),
    ]),
    'row4-w1': ((8, 128), [
        ('gemm_4bit_partial', (1, 8, 128, 256, 128, 64, 2, 2, 0), ['t']),
        ('reduce_partials', (1, 8, 128), BF, True),
    ]),
    'fused_forward_row-w1': ((8, 128), [
        ('slot', 0),
        ('gemm_4bit_partial', (1, 8, 128, 256, 128, 64, 2, 2, 0), [1000000]),
        ('barrier', 0),
        ('reduce_partials', (1, 8, 128), BF, True),
    ]),
    'fused_forward_row-refused-w1': ('gemm_4bit_partial does not serve this shard shape', [
        ('slot', 0),
        ('gemm_4bit_partial', (1, 8, 128, 256, 128, 64, 2, 2, 0), [1000000]),
    ]),
    'row8-refused-w1': ('the int8 GEMM does not serve this shard shape', [
        ('int8_row_stats', (8, 256), 0.0),
        ('int8_quant_with_stats', (8, 256), (8,), 0.0),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 256, 128, 0, 0), ['t']),
    ]),
    'fused_forward_row8-refused-w1': ('the int8 GEMM does not serve this shard shape', [
        ('int8_row_stats', (8, 256), 0.0),
        ('int8_quant_with_stats', (8, 256), (8,), 0.0),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 256, 128, 0, 0), [1000000]),
    ]),
    'col8-t0-w1': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 0.0),
        ('int8_gemm_multi_out', (0, 1, 8, 256, 128, 256, 2, 0), ['t']),
    ]),
    'fused_forward_col8-t0-w1': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 0.0),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 1, 8, 256, 128, 256, 2, 0), [1000000]),
        ('barrier', 0),
    ]),
    'row8-t0-w1': ((8, 128), [
        ('int8_row_stats', (8, 256), 0.0),
        ('int8_quant_with_stats', (8, 256), (8,), 0.0),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 256, 128, 0, 0), ['t']),
        ('int8_reduce_partials', (1, 8, 128), (8,), BF, None, None),
    ]),
    'fused_forward_row8-t0-w1': ((8, 128), [
        ('int8_row_stats', (8, 256), 0.0),
        ('int8_quant_with_stats', (8, 256), (8,), 0.0),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 256, 128, 0, 0), [1000000]),
        ('barrier', 0),
        ('int8_reduce_partials', (1, 8, 128), (8,), BF, None, None),
    ]),
    'col8-j2-w1': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 6.0),
        ('int8_outlier_prep', (2, 8, 8, 256, 128, 2, 0), None),
        ('int8_gemm_multi_out', (8, 1, 8, 256, 128, 256, 2, 0), ['t']),
    ]),
    'fused_forward_col8-j2-w1': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 6.0),
        ('slot', 0),
        ('int8_outlier_prep', (2, 8, 8, 256, 128, 2, 0), None),
        ('int8_gemm_multi_out', (8, 1, 8, 256, 128, 256, 2, 0), [1000000]),
        ('barrier', 0),
    ]),
    'row8-j2-w1': ((8, 128), [
        ('int8_row_stats', (8, 256), 6.0),
        ('int8_quant_with_stats', (8, 256), (8,), 6.0),
        ('int8_zero_columns', (2, 8, 256, 0), None),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 256, 128, 0, 0), ['t']),
        ('int8_outlier_prep', (2, 8, 8, 128, 256, 2, 0), None),
        ('int8_reduce_partials', (1, 8, 128), (8,), BF, (8, 8), (128, 8)),
    ]),
    'fused_forward_row8-j2-w1': ((8, 128), [
        ('int8_row_stats', (8, 256), 6.0),
        ('int8_quant_with_stats', (8, 256), (8,), 6.0),
        ('int8_zero_columns', (2, 8, 256, 0), None),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 256, 128, 0, 0), [1000000]),
        ('int8_outlier_prep', (2, 8, 8, 128, 256, 2, 0), None),
        ('barrier', 0),
        ('int8_reduce_partials', (1, 8, 128), (8,), BF, (8, 8), (128, 8)),
    ]),
    'col8-j65-w1': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 6.0),
        ('int8_gemm_multi_out', (0, 1, 8, 256, 128, 256, 2, 0), ['t']),
    ]),
    'fused_forward_col8-j65-w1': ((8, 256), [
        ('int8_vectorwise_quant', (8, 128), 6.0),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 1, 8, 256, 128, 256, 2, 0), ['t']),
        ('all_gather_into_tensor', (2048,), (2048,)),
        ('all_gather_into_tensor', (256, 65), (256, 65)),
        ('barrier', 0),
    ]),
    'row8-j65-w1': ((8, 128), [
        ('int8_row_stats', (8, 256), 6.0),
        ('int8_quant_with_stats', (8, 256), (8,), 6.0),
        ('int8_zero_columns', (65, 8, 256, 0), None),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 256, 128, 0, 0), ['t']),
        ('int8_outlier_prep', (65, 72, 8, 128, 256, 2, 0), None),
        ('int8_reduce_partials', (1, 8, 128), (8,), BF, None, None),
    ]),
    'fused_forward_row8-j65-w1': ((8, 128), [
        ('int8_row_stats', (8, 256), 6.0),
        ('int8_quant_with_stats', (8, 256), (8,), 6.0),
        ('int8_zero_columns', (65, 8, 256, 0), None),
        ('slot', 0),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 256, 128, 0, 0), [1000000]),
        ('int8_outlier_prep', (65, 72, 8, 128, 256, 2, 0), None),
        ('barrier', 0),
        ('int8_reduce_partials', (1, 8, 128), (8,), BF, None, None),
    ]),
    'col4-sp': ((8, 64), [
        ('all_gather_into_tensor', (8, 128), (2, 128)),
        ('gemm_4bit_strided', (8, 64, 128, 64, 64, 2, 2, 0), None),
    ]),
    'fused_forward_col_sp': ((8, 64), [
        ('slot', 0),
        ('copy', 0, 0, (2, 128), BF, 256),
        ('copy', 0, 1, (2, 128), BF, 256),
        ('copy', 0, 2, (2, 128), BF, 256),
        ('copy', 0, 3, (2, 128), BF, 256),
        ('barrier', 0),
        ('gemm_4bit_strided', (8, 64, 128, 64, 64, 2, 2, 0), None),
    ]),
    'row4-sp': ((2, 128), [
        ('gemm_4bit_partial', (1, 8, 128, 64, 128, 64, 2, 2, 0), ['t']),
        ('all_to_all_single', (4, 2, 128), (4, 2, 128)),
        ('reduce_partials', (4, 2, 128), BF, True),
    ]),
    'fused_forward_row_sp': ((2, 128), [
        ('slot', 0),
        ('gemm_4bit_partial_scatter', (4, 2, 8, 128, 64, 128, 64, 2, 2, 0), [1001024, 1011024, 1021024, 1031024]),
        ('barrier', 0),
        ('reduce_partials', (4, 2, 128), BF, True),
    ]),
    'fused_forward_row_sp-refused': ((2, 128), [
        ('slot', 0),
        ('gemm_4bit_partial_scatter', (4, 2, 8, 128, 64, 128, 64, 2, 2, 0), [1001024, 1011024, 1021024, 1031024]),
        ('gemm_4bit_partial', (1, 8, 128, 64, 128, 64, 2, 2, 0), ['t']),
        ('all_to_all_single', (4, 2, 128), (4, 2, 128)),
        ('barrier', 0),
        ('reduce_partials', (4, 2, 128), BF, True),
    ]),
    'fused_forward_row8_sp-refused': ((2, 128), [
        ('int8_row_stats', (8, 64), 0.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 0.0),
        ('slot', 0),
        ('int8_gemm_partial_scatter', (4, 2, 8, 128, 64, 128, 0), [1001024, 1011024, 1021024, 1031024]),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 64, 128, 0, 0), ['t']),
        ('all_to_all_single', (4, 2, 128), (4, 2, 128)),
        ('barrier', 0),
        ('int8_reduce_partials', (4, 2, 128), (2,), BF, None, None),
    ]),
    'col8-sp-t0': ((8, 64), [
        ('int8_vectorwise_quant_flags', (2, 128), 0.0),
        ('all_gather_into_tensor', (8, 128), (2, 128)),
        ('all_gather_into_tensor', (8,), (2,)),
        ('int8_gemm_multi_out', (0, 1, 8, 64, 128, 64, 2, 0), ['t']),
    ]),
    'fused_forward_col8_sp-t0': ((8, 64), [
        ('int8_vectorwise_quant_flags', (2, 128), 0.0),
        ('slot', 0),
        ('copy', 0, 0, (2, 128), I8, 256),
        ('copy', 0, 0, (2,), F32, 258),
        ('copy', 0, 1, (2, 128), I8, 256),
        ('copy', 0, 1, (2,), F32, 258),
        ('copy', 0, 2, (2, 128), I8, 256),
        ('copy', 0, 2, (2,), F32, 258),
        ('copy', 0, 3, (2, 128), I8, 256),
        ('copy', 0, 3, (2,), F32, 258),
        ('barrier', 0),
        ('int8_gemm_multi_out', (0, 1, 8, 64, 128, 64, 2, 0), ['t']),
    ]),
    'row8-sp-t0': ((2, 128), [
        ('int8_row_stats', (8, 64), 0.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 0.0),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 64, 128, 0, 0), ['t']),
        ('all_to_all_single', (4, 2, 128), (4, 2, 128)),
        ('int8_reduce_partials', (4, 2, 128), (2,), BF, None, None),
    ]),
    'fused_forward_row8_sp-t0': ((2, 128), [
        ('int8_row_stats', (8, 64), 0.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 0.0),
        ('slot', 0),
        ('int8_gemm_partial_scatter', (4, 2, 8, 128, 64, 128, 0), [1001024, 1011024, 1021024, 1031024]),
        ('barrier', 0),
        ('int8_reduce_partials', (4, 2, 128), (2,), BF, None, None),
    ]),
    'col8-sp-j2': ((8, 64), [
        ('int8_vectorwise_quant_flags', (2, 128), 6.0),
        ('all_reduce', (128,), I32),
        ('int8_zero_columns', (2, 2, 128, 0), None),
        ('int8_outlier_prep', (2, 8, 2, 64, 128, 2, 0), None),
        ('all_gather_into_tensor', (8, 128), (2, 128)),
        ('all_gather_into_tensor', (8,), (2,)),
        ('all_gather_into_tensor', (8, 8), (2, 8)),
        ('int8_gemm_multi_out', (8, 1, 8, 64, 128, 64, 2, 0), ['t']),
    ]),
    'fused_forward_col8_sp-j2': ((8, 64), [
        ('int8_vectorwise_quant_flags', (2, 128), 6.0),
        ('all_reduce', (128,), I32),
        ('int8_zero_columns', (2, 2, 128, 0), None),
        ('int8_outlier_prep', (2, 8, 2, 64, 128, 2, 0), None),
        ('slot', 0),
        ('copy', 0, 0, (2, 128), I8, 256),
        ('copy', 0, 0, (2,), F32, 258),
        ('copy', 0, 1, (2, 128), I8, 256),
        ('copy', 0, 1, (2,), F32, 258),
        ('copy', 0, 2, (2, 128), I8, 256),
        ('copy', 0, 2, (2,), F32, 258),
        ('copy', 0, 3, (2, 128), I8, 256),
        ('copy', 0, 3, (2,), F32, 258),
        ('barrier', 0),
        ('all_gather_into_tensor', (8, 8), (2, 8)),
        ('int8_gemm_multi_out', (8, 1, 8, 64, 128, 64, 2, 0), ['t']),
    ]),
    'row8-sp-j2': ((2, 128), [
        ('int8_row_stats', (8, 64), 6.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 6.0),
        ('int8_zero_columns', (2, 8, 64, 0), None),
        ('all_gather_into_tensor', (4,), (1,)),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 64, 128, 0, 0), ['t']),
        ('all_to_all_single', (4, 2, 128), (4, 2, 128)),
        ('int8_outlier_prep', (2, 8, 8, 128, 64, 2, 0), None),
        ('all_gather_into_tensor', (4352,), (1088,)),
        ('int8_reduce_partials', (4, 2, 128), (2,), BF, (2, 8), (128, 8)),
    ]),
    'fused_forward_row8_sp-j2': ((2, 128), [
        ('int8_row_stats', (8, 64), 6.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 6.0),
        ('int8_zero_columns', (2, 8, 64, 0), None),
        ('all_gather_into_tensor', (4,), (1,)),
        ('slot', 0),
        ('int8_gemm_partial_scatter', (4, 2, 8, 128, 64, 128, 0), [1001024, 1011024, 1021024, 1031024]),
        ('int8_outlier_prep', (2, 8, 8, 128, 64, 2, 0), None),
        ('all_gather_into_tensor', (4352,), (1088,)),
        ('barrier', 0),
        ('int8_reduce_partials', (4, 2, 128), (2,), BF, (2, 8), (128, 8)),
    ]),
    'col8-sp-j65': ((8, 64), [
        ('int8_vectorwise_quant_flags', (2, 128), 6.0),
        ('all_reduce', (128,), I32),
        ('int8_zero_columns', (65, 2, 128, 0), None),
        ('all_gather_into_tensor', (8, 128), (2, 128)),
        ('all_gather_into_tensor', (8,), (2,)),
        ('all_gather_into_tensor', (8, 65), (2, 65)),
        ('int8_gemm_multi_out', (0, 1, 8, 64, 128, 64, 2, 0), ['t']),
        ('all_gather_into_tensor', (2048,), (512,)),
        ('all_gather_into_tensor', (256, 65), (64, 65)),
    ]),
    'fused_forward_col8_sp-j65': ((8, 64), [
        ('int8_vectorwise_quant_flags', (2, 128), 6.0),
        ('all_reduce', (128,), I32),
        ('int8_zero_columns', (65, 2, 128, 0), None),
        ('slot', 0),
        ('copy', 0, 0, (2, 128), I8, 256),
        ('copy', 0, 0, (2,), F32, 258),
        ('copy', 0, 1, (2, 128), I8, 256),
        ('copy', 0, 1, (2,), F32, 258),
        ('copy', 0, 2, (2, 128), I8, 256),
        ('copy', 0, 2, (2,), F32, 258),
        ('copy', 0, 3, (2, 128), I8, 256),
        ('copy', 0, 3, (2,), F32, 258),
        ('barrier', 0),
        ('all_gather_into_tensor', (8, 65), (2, 65)),
        ('int8_gemm_multi_out', (0, 1, 8, 64, 128, 64, 2, 0), ['t']),
        ('all_gather_into_tensor', (2048,), (512,)),
        ('all_gather_into_tensor', (256, 65), (64, 65)),
    ]),
    'row8-sp-j65': ((2, 128), [
        ('int8_row_stats', (8, 64), 6.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 6.0),
        ('int8_zero_columns', (17, 8, 64, 0), None),
        ('all_gather_into_tensor', (4,), (1,)),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 64, 128, 0, 0), ['t']),
        ('all_gather_into_tensor', (4096,), (1024,)),
        ('int8_outlier_prep', (17, 24, 8, 128, 64, 2, 0), None),
        ('all_gather_into_tensor', (13056,), (3264,)),
        ('int8_reduce_partials', (4, 8, 128), (8,), BF, None, None),
    ]),
    'fused_forward_row8_sp-j65': ((2, 128), [
        ('int8_row_stats', (8, 64), 6.0),
        ('all_reduce', (8,), F32),
        ('int8_quant_with_stats', (8, 64), (8,), 6.0),
        ('int8_zero_columns', (17, 8, 64, 0), None),
        ('all_gather_into_tensor', (4,), (1,)),
        ('int8_gemm_multi_out', (0, 1, 8, 128, 64, 128, 0, 0), ['t']),
        ('all_gather_into_tensor', (4096,), (1024,)),
        ('int8_outlier_prep', (17, 24, 8, 128, 64, 2, 0), None),
        ('all_gather_into_tensor', (13056,), (3264,)),
        ('int8_reduce_partials', (4, 8, 128), (8,), BF, None, None),
    ]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_forward_events(monkeypatch, case):
    """Each forward issues exactly these events in this order, and returns this shape or raises this error."""
    assert _run(monkeypatch, case) == EVENTS[case]


@pytest.mark.parametrize("route", ["fused_forward", "fused_forward_col8"])
def test_gathered_column_routes_return_the_slot_and_alternate_slots(monkeypatch, route):
    """At inference the gathered column routes return their PeerGather slot itself; three calls take slots 0, 1, 0 and
    hand the GEMM the matching destinations."""
    w = World(monkeypatch, 4, 1)
    layer = _col4(w) if route == "fused_forward" else _col8(w, 0.0)
    peers = _gather(w)
    for step in range(3):
        assert getattr(par, route)(layer, _x(M, K), peers) is peers.bufs[step & 1]
    gemm = [e for e in w.log if e[0] in ("gemm_4bit_multi_out", "int8_gemm_multi_out")]
    assert [e for e in w.log if e[0] in ("slot", "barrier")] == [("slot", 0), ("barrier", 0), ("slot", 1),
                                                                   ("barrier", 1), ("slot", 0), ("barrier", 0)]
    assert [e[2] for e in gemm] == [w.ptrs(s, (N // 4) * 2) for s in (0, 1, 0)]


@pytest.mark.parametrize("route", ["fused_forward_row", "fused_forward_row_sp", "fused_forward_row8",
                                   "fused_forward_row8_sp"])
def test_row_routes_alternate_slots(monkeypatch, route):
    w = World(monkeypatch, 4, 1)
    sp, int8 = route.endswith("_sp"), "8" in route
    layer = _row8(w, 0.0, sp=sp) if int8 else _row4(w, sp=sp)
    peers = (_parts_sp if sp else _parts)(w, torch.int32 if int8 else torch.float32)
    for _ in range(3):
        getattr(par, route)(layer, _x(M, N // 4), peers)
    rows = M // 4 if sp else M
    dests = [e[2] for e in w.log if e[0] in ("gemm_4bit_partial", "gemm_4bit_partial_scatter", "int8_gemm_multi_out",
                                             "int8_gemm_partial_scatter")]
    assert [e for e in w.log if e[0] == "slot"] == [("slot", 0), ("slot", 1), ("slot", 0)]
    assert dests == [w.ptrs(s, rows * K * 4, own_first=not sp) for s in (0, 1, 0)]
