"""GPU parity: every non-grouped instance of the fused wgmma 4-bit GEMM, gemm4_tc_kernel<T, QT, MT, DQ, PART>.

112 instances serve every 4-bit GEMM of more than 8 tokens below the staged route's 2048: T = bf16 / fp16 (MT = 16,
32, 64, 128, 256) and T = float, the TF32 instance (MT <= 128); QT = NF4 / FP4; DQ = plain / nested statistics; PART
= the rounded T output / the fp32 partial.  Each call also picks a K split, a store path and its destinations.

a. Decoded weights, bit for bit, in every rounded 16-bit instance: identity activations (x = I_K, M = K tokens) make
   each output one exact product, out[m, n] = T(W_T[n, m] + bias[n]), where W_T is the library's blockwise
   dequantisation.  K = 64 (half a 128-deep stage), 192 and 576 (rows start mid-block and blocks begin mid-stage at
   blocksize >= 128), 1152 (past the 8-stage ring); blocksizes 32 to 4096; ragged N.
b. Every rounded 16-bit instance at the pair entry against the float64 oracle with forced K splits: 2, 3 over 5
   k-blocks (the last split short), the largest split that fits one wave, and the next one refused (return 100,
   before any launch).  Without a split the five token tiles agree bit for bit (the same k16 order), also on a
   problem with more tiles than SMs, where the persistent loop carries the ring across units.
c. Every partial instance through the dispatched entries, with and without the K split the rule picks (the
   256-token tile never splits): the partial against float64, T(partial + bias) equal to the same call's rounded
   output, and both equal to the pair entry at the rule's tile and split.
d. The rounded output to 2 and 8 destinations on the 16-byte and the element store paths, the partial to 3
   destinations, and the partial scattered over ranks whose row counts are not multiples of the tile.

The dispatched shapes are derived from the device's SM count with the rule of launch_gemm4_tc / launch_mt (restated
in tile_rule and split_of).  Every output starts NaN-filled, with padding columns and guard elements past its end;
an element stored outside [M, N] fails.  The bounds are the suite's: assert_close_to_exact (test_gpu_gemm4) for T
outputs, assert_partial_close (test_gpu_gemm4_cuda_core) for partials; the oracle is the C oracle up to 2^26
multiply-adds and float64 on the GPU over the decoded weights of (a) above that.

Which instance ran is proven from the kernel names, as in test_gpu_gemm4_cuda_core: one child process replays every
case's launches under torch.profiler and reports the template arguments of every 4-bit GEMM kernel it launched, and
each test asserts its own list.
"""
import ctypes as ct
import functools
import json
import re
import subprocess
import sys
from itertools import product
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import _native as nat
from tests.test_gpu_gemm4 import assert_close_to_exact, exact, make_problem
from tests.test_gpu_gemm4_cuda_core import QT_ARG, T_NAME, _arg, _instance, _profiled, assert_partial_close, case_key
from tests.test_gpu_gemm4_tf32 import make_problem as make_problem_tf32
from tests.test_gpu_gemm4_tf32 import rna_tf32

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
DT16 = ["bf16", "fp16"]
QTS = ["nf4", "fp4"]
DQS = [False, True]
TILES16 = [16, 32, 64, 128, 256]
TILES_TF32 = [16, 32, 64, 128]
TNAME = dict(T_NAME, tf32="float")  # "tf32": fp32 activations on the TF32 instance (dtype id 3)
STAGED_MIN_M = 2048                 # c_api.cu kStagedMinM: from here 16-bit calls take the staged route
MMA_MAX_M = 8                       # c_api.cu mma_max_m(): up to here 16-bit calls take the mma.sync decode kernel
C_ORACLE_MACS = 1 << 26             # larger problems: float64 on the GPU over the decoded weights
GUARD = 67                          # NaN elements after every output buffer
M_AT = {16: 15, 32: 27, 64: 63, 128: 100, 256: 1000}  # dispatched tokens per tile: rows_per_out 5, 9, 21, 25, 125
BLOCKSIZES = [32, 64, 128, 256, 4096]


def cdiv(a, b):
    return -(-a // b)


def instance(dtype, qt, mt, dq, part):
    """gemm4_tc_kernel<T, QT, MT, DQ, PART, GROUPED = false> as _tc_instance reports it."""
    return ("gemm4_tc_kernel", TNAME[dtype], QT_ARG[qt], str(mt), str(int(dq)), str(int(part)), "0")


def blocksize_of(mt, dq):
    return BLOCKSIZES[(TILES16.index(mt) + int(dq)) % len(BLOCKSIZES)]


# ------------------------------------------------------------------------ the tile and split rule (launch_gemm4_tc)
def tile_rule(M, N, dtype, sms):
    """The token tile launch_gemm4_tc picks: 16 / 32 / 64 up to that many tokens; then 256 (16-bit only) when the
    256-token tiles alone fill every SM, else 128."""
    if M <= 16:
        return 16
    if M <= 32:
        return 32
    if M <= 64:
        return 64
    if dtype != "tf32" and cdiv(M, 256) * cdiv(N, 128) >= sms:
        return 256
    return 128


def split_of(M, N, K, mt, dtype, sms, force=0):
    """(splits, stages per split) of launch_mt, force = the pair entry's force_splits (0: the rule, which splits when
    tiles * 2 <= SMs, by SMs / tiles, at least two stages per split); None where a forced split is refused because
    its tiles * splits do not fit one wave."""
    kb = cdiv(K, 64 if mt == 256 or dtype == "tf32" else 128)
    tiles = cdiv(M, mt) * cdiv(N, 128)
    if force == 0 and tiles * 2 > sms:
        return 1, kb
    v = force if force > 0 else sms // tiles
    v = max(1, min(v, kb if force > 0 else max(kb // 2, 1), 16))
    per = cdiv(kb, v)
    splits = cdiv(kb, per)
    if splits > 1 and tiles * splits > sms:
        return None
    return splits, per


def dispatched_shape(mt, split, dtype, sms, M=None):
    """(M, N, K) that the dispatched entries send to token tile mt, with the rule's K split or without one.  N is
    ragged (N % 8 == 3, a partial last 128-feature tile); without a split N is wide enough that tiles * 2 > SMs."""
    M = M_AT[mt] if M is None else M
    if split:
        N, K = 203, 1152
    else:
        K = 320
        nt = cdiv(sms, cdiv(M, 256)) if mt == 256 else sms // (2 * cdiv(M, mt)) + 1
        N = 128 * nt - 37
    splits, _ = split_of(M, N, K, mt, dtype, sms)
    if tile_rule(M, N, dtype, sms) != mt or (splits > 1) != split or not MMA_MAX_M < M < STAGED_MIN_M:
        raise ValueError(f"({M}, {N}, {K}) does not take tile {mt} {'with' if split else 'without'} a split")
    return M, N, K


# ------------------------------------------------------------------------------------------ buffers and C entries
def out_buffer(rows, ldc, dtype, off=0):
    """A NaN-filled [rows, ldc] output `off` elements into its allocation, with GUARD NaN elements after it."""
    buf = torch.full((off + rows * ldc + GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf[off:off + rows * ldc].view(rows, ldc)


def inside(t, N):
    """t[:, :N], after asserting that nothing else of t's allocation (offset, padding columns, guard) was stored."""
    whole = torch.empty(0, dtype=t.dtype, device=t.device).set_(t.untyped_storage())
    keep = torch.ones(whole.numel(), dtype=torch.bool, device=t.device)
    rows = torch.arange(t.shape[0], device=t.device)[:, None] * t.stride(0)
    keep[(t.storage_offset() + rows + torch.arange(N, device=t.device)[None, :]).view(-1)] = False
    assert torch.isnan(whole[keep]).all(), "stored outside [M, N]"
    return t[:, :N]


def bits(t):
    t = t.contiguous()
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def tdtype(dtype):
    return torch.float32 if dtype == "tf32" else nat.DTYPE[dtype]


def dtype_id(dtype):
    return 3 if dtype == "tf32" else nat.DTYPE_ID[dtype]


def _operands(p):
    return (nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
            nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]))


def _ptrs(outs):
    return ct.cast((ct.c_void_p * len(outs))(*[o.data_ptr() for o in outs]), ct.c_void_p)


def pair(p, out, mt, splits):
    """The developer entry: the rounded instance at token tile mt, force_splits = splits.  Returns its code."""
    return nat.lib.cbnb_b200_gemm_4bit_pair(
        *_operands(p), out.data_ptr(), nat.ptr(p["bias"]), p["M"], p["N"], p["K"], out.stride(0), p["bs"],
        nat.QT_ID[p["qt"]], dtype_id(p["dtype"]), mt, splits, None, nat.stream())


def strided(p, out):
    nat.lib.cbnb_b200_gemm_4bit_strided(
        *_operands(p), out.data_ptr(), nat.ptr(p["bias"]), p["M"], p["N"], p["K"], out.stride(0), p["bs"],
        nat.QT_ID[p["qt"]], dtype_id(p["dtype"]), nat.stream())


def multi_out(p, outs):
    return nat.lib.cbnb_b200_gemm_4bit_multi_out(
        *_operands(p), _ptrs(outs), len(outs), nat.ptr(p["bias"]), p["M"], p["N"], p["K"], outs[0].stride(0),
        p["bs"], nat.QT_ID[p["qt"]], dtype_id(p["dtype"]), nat.stream())


def partial(p, outs):
    return nat.lib.cbnb_b200_gemm_4bit_partial(
        *_operands(p), _ptrs(outs), len(outs), p["M"], p["N"], p["K"], outs[0].stride(0), p["bs"],
        nat.QT_ID[p["qt"]], dtype_id(p["dtype"]), nat.stream())


def partial_scatter(p, outs):
    return nat.lib.cbnb_b200_gemm_4bit_partial_scatter(
        *_operands(p), _ptrs(outs), len(outs), outs[0].shape[0], p["M"], p["N"], p["K"], outs[0].stride(0),
        p["bs"], nat.QT_ID[p["qt"]], dtype_id(p["dtype"]), nat.stream())


def finish():
    torch.cuda.synchronize()
    nat.check()


# ---------------------------------------------------------------------------------------------------- references
def weights(p):
    """W_T [N, K] as F.dequantize_4bit decodes it: the library's blockwise dequantisation with the scale it uses
    (nested: the dequantised 8-bit absmax plus the offset, two roundings)."""
    scale = p["absmax"]
    if p["absmax_8bit"] is not None:
        nb = p["absmax_8bit"].numel()
        scale = nat.dequantize(nat.lib, p["absmax_8bit"], p["absmax"], 256, nb, None, p["absmax_code"], "fp32")
        scale = scale + p["absmax_offset"]
    W = nat.dequantize(nat.lib, p["packed"], scale.contiguous(), p["bs"], p["N"] * p["K"], p["qt"], None, p["dtype"])
    return W.view(p["N"], p["K"])


def reference(p, bias=True):
    """The float64 [M, N] result (numpy) of a 16-bit problem: the C oracle up to C_ORACLE_MACS multiply-adds, above
    that float64 on the GPU over weights(p), which test a proves to be the kernel's decoded weights bit for bit."""
    q = p if bias else dict(p, bias=None)
    if p["M"] * p["N"] * p["K"] <= C_ORACLE_MACS:
        return exact(q)
    y = q["x"].double() @ weights(q).double().t()
    if q["bias"] is not None:
        y += q["bias"].double()
    return y.cpu().numpy()


def reference_tf32(p):
    """The float64 partial of a TF32 problem (TF32-exact activations): every product with rna_tf32(W32) is exact."""
    return (p["x"].double() @ rna_tf32(p["W32"]).double().t()).cpu().numpy()


# ------------------------------------------------------------------------ the launches of each case (seeded inputs)
KS_DECODE = [64, 192, 576, 1152]  # half a stage; lowest set bit 64 (twice); nine 128-deep stages, past the ring
N_DECODE = 203


@functools.lru_cache(maxsize=None)
def decode_problem(dtype, qt, dq, K, bs, bias):
    p = make_problem(1, N_DECODE, K, qt, dtype, bs=bs, nested=dq, bias=bias, seed=K + bs)
    p.update(M=K, x=torch.eye(K, dtype=nat.DTYPE[dtype], device="cuda"))
    return p


def decode_runs():
    """(K, blocksize, bias) of every decode launch: bias on every other one, so each K and blocksize has both."""
    return [(K, bs, (i + j) % 2 == 1) for i, K in enumerate(KS_DECODE) for j, bs in enumerate(BLOCKSIZES)]


def launch_decode(a):
    runs = []
    for K, bs, bias in decode_runs():
        p = decode_problem(a["dtype"], a["qt"], a["dq"], K, bs, bias)
        out = out_buffer(K, N_DECODE + 5, nat.DTYPE[a["dtype"]])
        assert pair(p, out, a["mt"], 1) == 0, (K, bs)
        runs.append((p, out))
    finish()
    return runs


def launch_tiles(a):
    """The five tiles without a split on a problem with bias and on one with more tiles than SMs at every tile."""
    res = []
    for M, N, K, bias, seed in [(100, 203, 640, True, 41), (1000, a["n_big"], 384, False, 42)]:
        p = make_problem(M, N, K, a["qt"], a["dtype"], bs=a["bs"], nested=a["dq"], bias=bias, seed=seed)
        outs = [out_buffer(M, N + 5, nat.DTYPE[a["dtype"]]) for _ in TILES16]
        for mt, o in zip(TILES16, outs):
            assert pair(p, o, mt, 1) == 0, mt
        res.append((p, outs))
    finish()
    return res


def launch_splits(a):
    """Forced splits 2 and 3 of 5 (10 at the 256-token tile's 64-deep stages) k-blocks, with bias; the largest split
    of one wave and the next, refused one, without."""
    dt, mt = a["dtype"], a["mt"]
    p1 = make_problem(100, 203, 640, a["qt"], dt, bs=a["bs"], nested=a["dq"], bias=True, seed=41)
    p2 = make_problem(150, 203, 2048, a["qt"], dt, bs=a["bs"], nested=a["dq"], bias=False, seed=43)
    o2, o3 = out_buffer(100, 208, nat.DTYPE[dt]), out_buffer(100, 208, nat.DTYPE[dt])
    ow, over = out_buffer(150, 208, nat.DTYPE[dt]), out_buffer(150, 208, nat.DTYPE[dt])
    assert pair(p1, o2, mt, 2) == 0 and pair(p1, o3, mt, 3) == 0
    assert pair(p2, ow, mt, a["wave"]) == 0
    rc_over = pair(p2, over, mt, a["over"]) if a["over"] else None
    finish()
    return p1, o2, o3, p2, ow, over, rc_over


def _problem(a):
    M, N, K = a["shape"]
    if a["dtype"] == "tf32":
        p = make_problem_tf32(M, N, K, a["qt"], a["bs"], a["dq"], True, seed=44)
        p["dtype"] = "tf32"
        return p
    return make_problem(M, N, K, a["qt"], a["dtype"], bs=a["bs"], nested=a["dq"], bias=True, seed=44)


def launch_partial(a):
    """The dispatched rounded and partial entries, then the pair entry at the rule's tile and split."""
    p = _problem(a)
    M, N = p["M"], p["N"]
    out, pair_out = out_buffer(M, N + 5, tdtype(a["dtype"])), out_buffer(M, N + 5, tdtype(a["dtype"]))
    part = out_buffer(M, N + 5, torch.float32)
    strided(p, out)
    assert partial(p, [part]) == 0
    assert pair(p, pair_out, a["mt"], a["splits"]) == 0
    finish()
    return p, out, part, pair_out


def launch_dests(a):
    """The single-destination call, _multi_out to 2 (16-byte stores), 8 (odd ldc) and 2 (one base an element off)
    destinations, _partial to 3 destinations and to 1, and _partial_scatter over a["ranks"] ranks."""
    p = _problem(a)
    M, N, T = p["M"], p["N"], nat.DTYPE[a["dtype"]]
    ld8 = N + 5  # N % 8 == 3: a multiple of 8, so the 16-byte path, with a tail at the last 3 features
    plain = out_buffer(M, N, T)
    vec = [out_buffer(M, ld8, T) for _ in range(2)]
    odd = [out_buffer(M, N + 2, T) for _ in range(8)]
    off = [out_buffer(M, ld8, T), out_buffer(M, ld8, T, off=1)]
    parts = [out_buffer(M, ld8, torch.float32) for _ in range(3)]
    single = out_buffer(M, N, torch.float32)
    scat = [out_buffer(M // a["ranks"], N + 2, torch.float32) for _ in range(a["ranks"])]
    strided(p, plain)
    rcs = [multi_out(p, vec), multi_out(p, odd), multi_out(p, off), partial(p, parts), partial(p, [single]),
           partial_scatter(p, scat)]
    finish()
    return p, rcs, plain, vec + odd + off, parts, single, scat


LAUNCHERS = {"decode": launch_decode, "tiles": launch_tiles, "splits": launch_splits, "partial": launch_partial,
             "dests": launch_dests}


def launch(case):
    kind, a = case
    return LAUNCHERS[kind](a)


# ------------------------------------------------------------------------------------------------ the case table
def decode_case(dtype, qt, dq, mt):
    return ["decode", dict(dtype=dtype, qt=qt, dq=dq, mt=mt)]


def tiles_case(dtype, qt, dq, sms):
    nt = sms // 4 + 1  # 1000 tokens: 4 256-token tiles per 128 features, 4 * nt > SMs
    return ["tiles", dict(dtype=dtype, qt=qt, dq=dq, bs=64 if dq else 128, n_big=128 * nt - 37)]


def splits_case(dtype, qt, dq, mt, sms):
    wave = max(f for f in range(1, 17) if split_of(150, 203, 2048, mt, dtype, sms, force=f) is not None)
    over = next((f for f in range(wave + 1, 17) if split_of(150, 203, 2048, mt, dtype, sms, force=f) is None), 0)
    return ["splits", dict(dtype=dtype, qt=qt, dq=dq, mt=mt, bs=blocksize_of(mt, dq), wave=wave, over=over)]


def partial_case(dtype, qt, dq, mt, split, sms):
    shape = dispatched_shape(mt, split, dtype, sms)
    splits, per = split_of(*shape, mt, dtype, sms)
    assert split_of(*shape, mt, dtype, sms, force=splits) == (splits, per)  # the pair entry runs the same units
    return ["partial", dict(dtype=dtype, qt=qt, dq=dq, mt=mt, bs=blocksize_of(mt, dq), shape=list(shape),
                            splits=splits)]


DEST_RANKS = {16: 3, 32: 3, 64: 3, 128: 4, 256: 8}


def dests_case(mt, split, sms):
    i = 2 * TILES16.index(mt) + int(split)
    dtype, qt, dq = DT16[i % 2], QTS[(i // 2) % 2], i % 3 == 0
    shape = dispatched_shape(mt, split, dtype, sms)
    splits, _ = split_of(*shape, mt, dtype, sms)
    return ["dests", dict(dtype=dtype, qt=qt, dq=dq, mt=mt, bs=blocksize_of(mt, dq), shape=list(shape),
                          splits=splits, ranks=DEST_RANKS[mt])]


PARTIAL_ROWS = ([(dt, qt, dq, mt, s) for dt, qt, dq, mt in product(DT16, QTS, DQS, TILES16)
                 for s in ([False] if mt == 256 else [False, True])]
                + [("tf32", qt, dq, mt, s) for qt, dq, mt, s in product(QTS, DQS, TILES_TF32, [False, True])])
DEST_ROWS = [(mt, s) for mt in TILES16 for s in ([False] if mt == 256 else [False, True])]


def all_cases(sms):
    """The case of every test of this file for a device of `sms` SMs, in the order the child replays them."""
    cases = [decode_case(*r) for r in product(DT16, QTS, DQS, TILES16)]
    cases += [tiles_case(*r, sms) for r in product(DT16, QTS, DQS)]
    cases += [splits_case(*r, sms) for r in product(DT16, QTS, DQS, TILES16)]
    cases += [partial_case(*r, sms) for r in PARTIAL_ROWS]
    cases += [dests_case(*r, sms) for r in DEST_ROWS]
    return cases


def expected(case, sms):
    """[(instance, K splits)] of every gemm4_tc_kernel launch of the case, in launch order."""
    kind, a = case
    if kind == "tiles":
        return [(instance(a["dtype"], a["qt"], mt, a["dq"], 0), 1) for mt in TILES16] * 2
    inst = functools.partial(instance, a["dtype"], a["qt"], a["mt"], a["dq"])
    if kind == "decode":
        return [(inst(0), 1)] * len(decode_runs())
    if kind == "splits":
        forced = [(100, 203, 640, 2), (100, 203, 640, 3), (150, 203, 2048, a["wave"])]
        return [(inst(0), split_of(M, N, K, a["mt"], a["dtype"], sms, force=f)[0]) for M, N, K, f in forced]
    if kind == "partial":
        return [(inst(0), a["splits"]), (inst(1), a["splits"]), (inst(0), a["splits"])]
    return [(inst(0), a["splits"])] * 4 + [(inst(1), a["splits"])] * 3  # dests


# ----------------------------------------------------------------------- the launch record (a profiled child)
def _tc_instance(name: str):
    """(kernel, T, QT, MT, DQ, PART, GROUPED) of a gemm4_tc_kernel name; any other 4-bit GEMM kernel as
    test_gpu_gemm4_cuda_core reports it; None for every other kernel."""
    m = re.search(r"(gemm4_tc_kernel)<([^<>]*)>", name)
    if m:
        return [m.group(1)] + [_arg(x) for x in m.group(2).split(",")]
    return _instance(name)


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def record_launches_main():
    """The child: reads a JSON list of cases on stdin and prints one line "LAUNCHES <json>" mapping each case's key to
    the 4-bit GEMM kernel instances it launched (None: the profiler recorded no kernels; a string: the error)."""
    cases = json.loads(sys.stdin.read())
    for _ in range(5):  # the first sessions of a process can record nothing while the profiler starts up
        if _profiled(lambda: torch.ones(1, device="cuda").mul_(2)):
            break
    record = {}
    for case in cases:
        got = None
        try:
            for _ in range(2):
                kernels = _profiled(lambda: launch(case))
                if kernels:
                    got = [i for i in (_tc_instance(e.name) for e in kernels) if i is not None]
                    break
        except Exception as e:  # reported by the test of this case
            got = f"{type(e).__name__}: {e}"
        record[case_key(case)] = got
    print("LAUNCHES " + json.dumps(record), flush=True)


@pytest.fixture(scope="module")
def launches():
    """{case key: the instances its launches ran}, recorded once for every test of this file by the profiled child."""
    code = (f"import sys; sys.path.insert(0, {str(ROOT)!r}); "
            "from tests.test_gpu_gemm4_wgmma_instances import record_launches_main; record_launches_main()")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], input=json.dumps(all_cases(sm_count())),
                       capture_output=True, text=True, cwd=str(ROOT), timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("LAUNCHES ")]
    if r.returncode != 0 or not lines:
        pytest.fail(f"the profiled child exited with {r.returncode}:\n{r.stderr[-4000:]}")
    return json.loads(lines[-1][len("LAUNCHES "):])


def assert_ran(launches, case):
    """The case's recorded instances are its table entry's; skips (only this last assertion) without a record."""
    got = launches[case_key(case)]
    if got is None:
        pytest.skip("torch.profiler recorded no CUDA kernels here: which kernel instance ran is not confirmed")
    assert not isinstance(got, str), f"the profiled replay of this case failed: {got}"
    assert [tuple(i) for i in got] == [i for i, _ in expected(case, sm_count())]


# --------------------------------------------------------------------- a. decoded weights, every rounded instance
@pytest.mark.parametrize("mt", TILES16)
@pytest.mark.parametrize("dq", DQS, ids=["plain", "nested"])
@pytest.mark.parametrize("qt", QTS)
@pytest.mark.parametrize("dtype", DT16)
def test_decoded_weights_bit_for_bit(launches, dtype, qt, dq, mt):
    """x = I_K: out[m, n] = T(W_T[n, m] + bias[n]), one exact product per output, W_T the library's dequantisation.
    Without bias the expected value is W_T + 0.0: FP4's -0 code decodes to -0 and the accumulator, which starts at +0,
    turns it into +0."""
    case = decode_case(dtype, qt, dq, mt)
    for p, out in launch(case):
        got = inside(out, N_DECODE)
        want = weights(p).t().float() + (p["bias"].float() if p["bias"] is not None else 0.0)
        bad = bits(got) != bits(want.to(got.dtype))
        assert not bad.any(), f"K={p['K']} blocksize={p['bs']}: {int(bad.sum())} decoded weights differ"
    assert_ran(launches, case)


# ------------------------------------------------------------------ b. every rounded 16-bit instance, forced splits
@pytest.mark.parametrize("dq", DQS, ids=["plain", "nested"])
@pytest.mark.parametrize("qt", QTS)
@pytest.mark.parametrize("dtype", DT16)
def test_tiles_agree_without_a_split(launches, dtype, qt, dq):
    """Without a K split every token tile sums the same k16 steps in the same order: the five tiles agree bit for
    bit, with bias, and on 1000 tokens whose tiles outnumber the SMs at every tile (the persistent loop carries the
    ring from unit to unit), and meet the oracle bound."""
    case = tiles_case(dtype, qt, dq, sm_count())
    for p, outs in launch(case):
        got = [inside(o, p["N"]) for o in outs]
        for mt, g in zip(TILES16[1:], got[1:]):
            assert torch.equal(bits(g), bits(got[0])), f"tiles {mt} and 16 disagree"
        assert_close_to_exact(got[0], reference(p), dtype, p["K"])
    assert_ran(launches, case)


@pytest.mark.parametrize("mt", TILES16)
@pytest.mark.parametrize("dq", DQS, ids=["plain", "nested"])
@pytest.mark.parametrize("qt", QTS)
@pytest.mark.parametrize("dtype", DT16)
def test_forced_k_splits(launches, dtype, qt, dq, mt):
    """Forced splits 2 and 3 (uneven: 2, 2, 1 k-blocks; 4, 4, 2 at the 256-token tile), and the largest split whose
    tiles fit one wave, against the oracle; one split more is refused with 100 before any launch."""
    sms = sm_count()
    case = splits_case(dtype, qt, dq, mt, sms)
    p1, o2, o3, p2, ow, over, rc_over = launch(case)
    y1 = reference(p1)
    for o in (o2, o3):
        assert_close_to_exact(inside(o, 203), y1, dtype, p1["K"])
    assert_close_to_exact(inside(ow, 203), reference(p2), dtype, p2["K"])
    if case[1]["over"]:
        assert rc_over == 100 and torch.isnan(over).all()
    assert [s for _, s in expected(case, sms)][:2] == [2, 3]
    assert_ran(launches, case)


# --------------------------------------------------------------------------- c. every partial instance, dispatched
@pytest.mark.parametrize("dtype,qt,dq,mt,split", [
    pytest.param(*r, id=f"{r[0]}-{r[1]}-{'nested' if r[2] else 'plain'}-MT{r[3]}-{'split' if r[4] else 'nosplit'}")
    for r in PARTIAL_ROWS])
def test_partial_instance(launches, dtype, qt, dq, mt, split):
    """_partial on a shape the rule sends to tile mt: the fp32 partial meets the float64 bound; T(partial + bias) is
    the same call's rounded output (_strided) bit for bit; and the pair entry at the rule's tile and split gives that
    output too, which proves which split ran."""
    case = partial_case(dtype, qt, dq, mt, split, sm_count())
    p, out, part, pair_out = launch(case)
    N, K = p["N"], p["K"]
    got, pg, pr = inside(out, N), inside(part, N), inside(pair_out, N)
    if dtype == "tf32":
        assert_partial_close(pg, reference_tf32(p), K)
    else:
        assert_partial_close(pg, reference(p, bias=False), K)
        assert_close_to_exact(got, reference(p), dtype, K)
    assert torch.equal(bits((pg + p["bias"].float()).to(got.dtype)), bits(got))
    assert torch.equal(bits(pr), bits(got))
    assert_ran(launches, case)


# ---------------------------------------------------------------------------------- d. destinations, store paths
@pytest.mark.parametrize("mt,split", [pytest.param(*r, id=f"MT{r[0]}-{'split' if r[1] else 'nosplit'}")
                                      for r in DEST_ROWS])
def test_destinations_and_store_paths(launches, mt, split):
    """Every destination of _multi_out holds the single-destination output bit for bit, on the 16-byte store path
    (aligned bases, ldc % 8 == 0, N % 8 != 0) and on the element path (odd ldc; one base an element off); every
    destination of _partial holds the single-destination partial; _partial_scatter gives each rank its rows of it,
    with rows_per_out not a multiple of the tile, so that one tile spans two ranks."""
    case = dests_case(mt, split, sm_count())
    p, rcs, plain, copies, parts, single, scat = launch(case)
    N, K = p["N"], p["K"]
    assert rcs == [0] * len(rcs)
    want = inside(plain, N)
    assert_close_to_exact(want, reference(p), p["dtype"], K)
    for i, o in enumerate(copies):
        assert torch.equal(bits(inside(o, N)), bits(want)), f"destination {i}"
    one = inside(single, N)
    assert torch.equal(bits((one + p["bias"].float()).to(want.dtype)), bits(want))
    for i, o in enumerate(parts):
        assert torch.equal(bits(inside(o, N)), bits(one)), f"partial destination {i}"
    r = scat[0].shape[0]
    assert r % mt != 0
    for s, o in enumerate(scat):
        assert torch.equal(bits(inside(o, N)), bits(one[s * r:(s + 1) * r])), f"rank {s}"
    assert_ran(launches, case)
