"""GPU parity: every blockwise quantize and dequantize kernel instance, over several grid-stride rounds, against the
CPU oracle and (where it serves the case) the reference CUDA library; the nested-statistics decoders at scale; the
edges where flush-to-zero arithmetic decides the result; and the blocksizes the entries refuse.

The persistent kernels cap their grid and loop (blockwise.cu):

=========================================  =========================================  ===========================
kernel                                     one grid-stride round                      grid cap
=========================================  =========================================  ===========================
quantize_blockwise_kernel                  grid x kQThreads x kQEPT = 4096 elements     8 S CTAs
quantize_blockwise_generic_kernel          grid x 8 warps, one quant block per warp     8 S CTAs
dequantize_blockwise_kernel                grid x kDqThreads x kDqUnroll 16-byte vectors 8 S CTAs
dequantize4_prmt_kernel                    grid x kD4Warps x 32 units of 64 elements    4 S CTAs
dequantize_blockwise_generic_kernel        grid x 256 elements                          8 S CTAs
=========================================  =========================================  ===========================

S is the device's multi_processor_count, and every size below is computed from it.  Each test asserts the round count
that its size gives under those constants, and the grid that the profiler recorded for each launch (the chrome-trace
export of torch.profiler carries it), so a change of the launch constants fails here instead of silently shrinking a
test to one round.

Which instance ran is proven from the kernel names, as in test_gpu_gemm4_cuda_core: each test's launches are a function
of JSON arguments and seeded inputs (a build step that makes the inputs, then the launches), and one child process
(the same interpreter, which exits when done) replays every case with only the launches under torch.profiler and
reports each blockwise kernel's demangled name, template arguments and grid.  QT prints as 0 (8-bit, the reference's
7-step code walk), 3 (8-bit, the bracket-table search), 1 (FP4) or 2 (NF4).  A second child runs with
BNB_B200_Q8_WALK=1 (read once per process) and reports a SHA-256 of every 8-bit quantize case's guarded outputs: they
equal the bracket search's bytes.  If the profiler records nothing, only that assertion is skipped.

==============================================  ================================================================
instance                                        test
==============================================  ================================================================
quantize_blockwise_kernel<T, 3 | 1 | 2>         test_quantize_fast_path_rounds
quantize_blockwise_kernel<T, 0>                 test_quantize_walk_equals_bracket_search (the walk child)
quantize_blockwise_generic_kernel<T, QT>        test_quantize_fast_path_rounds (tail), test_quantize_generic_routes
dequantize4_prmt_kernel<T16, QT, false>         test_dequantize_rounds (prmt rows)
dequantize_blockwise_kernel<T, 0>               test_dequantize_rounds (8-bit rows)
dequantize_blockwise_kernel<float, QT>          test_dequantize_rounds (4-bit fp32 rows)
dequantize_blockwise_kernel<T16, QT>            test_dequantize_rounds (codes + 8 bytes, blocksize 16)
dequantize_blockwise_generic_kernel<T, QT>      test_dequantize_rounds (tails), test_dequantize_generic_routes
dequantize4_prmt_kernel<T16, QT, true>          test_nested_panel_decode
==============================================  ================================================================

Every output buffer carries a guard region past its end (quantize: codes and absmax; dequantize: the output, filled
with NaN), which must keep its fill.  Bars: absmax and dequantized values bit for bit against the oracle (fp32 compared
as bits), codes against the oracle with the threshold-adjacent allowance of test_gpu_blockwise, and everything bit for
bit against the reference CUDA library where it serves the case (power-of-two blocksizes; quantize 32..4096, 8-bit from
64; dequantize 8-bit from 64, 4-bit from 32).  The reference comparison comes last in each test: without the reference
build it is skipped, visibly.

Edges (test_quantize_edges / test_dequantize_edges).  The kernels flush subnormals in every multiply, absolute value
and max (mul.ftz, abs.ftz, max.ftz, rcp.approx.ftz), as the reference built with fast math does.  On an H100 the
kernels did the following; absmax is asserted directly, the codes as equal to the reference CUDA kernel's:

* a block whose |x| are all subnormal has absmax 0: its codes are those of NaN (0 * rcp(0) = 0 * inf);
* a block with max |x| >= 2^126 has a subnormal reciprocal, flushed to 0: every finite element gets the code of 0.0;
* +-inf in a block: absmax = inf, rcp(inf) = 0, the finite elements get the code of 0.0 and the inf the code of NaN;
* one NaN in a block: max.ftz ignores it, absmax is the maximum of the rest, the NaN gets the code of NaN;
* an all-NaN block: absmax stays at the starting value -FLT_MAX and every element gets the code of NaN;
* dequantize: value * absmax with a subnormal absmax or a subnormal product flushed to a zero of the product's sign,
  rounded once to T (bf16 has subnormals of its own, so it tells a flushed product from an IEEE one).
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from tests import _native as nat
from tests.test_gpu_blockwise import _check_codes_vs_oracle, _code, _inputs
from tests.test_gpu_gemm4_cuda_core import _arg, at_offset

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
T_NAME = {"bf16": "__nv_bfloat16", "fp16": "__half", "fp32": "float"}
QT_ARG = {None: "3", "fp4": "1", "nf4": "2"}  # the 8-bit quantizer's default instance is the bracket search (3)
DQ_QT_ARG = {None: "0", "fp4": "1", "nf4": "2"}
GUARD = 64  # bytes / elements of guard region past every output
SENTINEL_BYTE = 0xA5
SENTINEL_F32 = 0x7F81DEAD  # a signalling-NaN bit pattern no kernel writes

# launch constants of blockwise.cu
Q_TILE, Q_CAP = 256 * 16, 8      # kQThreads x kQEPT elements per tile; grid <= 8 S
QG_WARPS, QG_CAP = 8, 8          # the generic quantizer: one block per warp, 8 warps per CTA; grid <= 8 S
DQ_VECS, DQ_CAP = 256 * 8, 8     # kDqThreads x kDqUnroll vectors per CTA; grid <= 8 S
D4_UNITS, D4_CAP = 8 * 32, 4     # kD4Warps x 32 units of 64 elements per CTA; grid <= 4 S
DG_ELEMS, DG_CAP = 256, 8        # the generic dequantizer: one element per thread; grid <= 8 S


def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def cdiv(a, b):
    return -(-a // b)


def capped(want, cap):
    return min(want, cap * sms())


def rounds(work, grid, per_cta):
    return cdiv(work, grid * per_cta)


def sync():
    torch.cuda.synchronize()


def f32_bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().contiguous().cpu().view(torch.int32).numpy().view(np.uint32)


def out_bits(t: torch.Tensor) -> np.ndarray:
    return f32_bits(t) if t.dtype == torch.float32 else nat.to_bits(t)


def digest(tensors) -> str:
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


# ------------------------------------------------------------------------------- guarded calls of the C entries
def quantize_guarded(L, A, bs, qt, dtype, code):
    """The reference-ABI quantize entry into codes / absmax buffers that run GUARD bytes / floats past the end, the
    guards filled with sentinels.  Returns (codes buffer, absmax buffer), guards included."""
    n = A.numel()
    nbytes = n if qt is None else (n + 1) // 2
    codes = torch.full((nbytes + GUARD,), SENTINEL_BYTE, device="cuda", dtype=torch.uint8)
    absmax = torch.empty(cdiv(n, bs) + GUARD, device="cuda", dtype=torch.float32)
    absmax.view(torch.int32).fill_(SENTINEL_F32)
    fn = getattr(L, f"cquantize_blockwise_{dtype}" + ("" if qt is None else f"_{qt}"))
    sync()
    fn(nat.ptr(code), A.data_ptr(), absmax.data_ptr(), codes.data_ptr(), bs, n)
    sync()
    return codes, absmax


def assert_quantize_guards(codes, absmax, n, bs, qt):
    nbytes = n if qt is None else (n + 1) // 2
    assert (codes[nbytes:] == SENTINEL_BYTE).all(), "codes written past the end"
    assert (f32_bits(absmax[cdiv(n, bs):]) == SENTINEL_F32).all(), "absmax written past the end"


def dequantize_guarded(L, codes, absmax, bs, n, qt, dtype, code, out_off=0):
    """The dequantize entry into an output `out_off` elements past a NaN-filled buffer's start, GUARD elements of NaN
    past its end.  Returns the whole buffer."""
    buf = torch.full((out_off + n + GUARD,), float("nan"), device="cuda", dtype=nat.DTYPE[dtype])
    out = buf[out_off:out_off + n]
    fn = getattr(L, f"cdequantize_blockwise_{dtype}" + ("" if qt is None else f"_{qt}"))
    sync()
    fn(nat.ptr(code), codes.data_ptr(), absmax.data_ptr(), out.data_ptr(), bs, n, nat.stream())
    sync()
    return buf


def assert_dequantize_guards(buf, n, out_off):
    fill = out_bits(torch.full((1,), float("nan"), dtype=buf.dtype))[0]
    bits = out_bits(buf)
    assert (bits[:out_off] == fill).all() and (bits[out_off + n:] == fill).all(), "output written outside [0, n)"


def check_dequantized(got_bits, want_bits, what=""):
    bad = np.nonzero(got_bits != want_bits)[0]
    assert bad.size == 0, (f"{bad.size} {what} outputs differ from the oracle; first at {bad[:8].tolist()}: "
                           f"{got_bits[bad[:8]].tolist()} != {want_bits[bad[:8]].tolist()}")


# ----------------------------------------------------------------------------------- the launches of each test
def build_quantize(dtype, qt, n, bs, a_off=0):
    """Seeded activations (tests.test_gpu_blockwise._inputs) `a_off` elements past an allocation's start."""
    A = _inputs(n, dtype)
    if a_off:
        A = at_offset(A, a_off)
    code = _code() if qt is None else None
    return dict(A=A, code=code), lambda: quantize_guarded(nat.lib, A, bs, qt, dtype, code)


def _dequantize_inputs(n, bs, qt, seed, codes_off):
    g = torch.Generator(device="cpu").manual_seed(seed)
    nbytes = n if qt is None else (n + 1) // 2
    codes = torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8).cuda()
    if codes_off:
        codes = at_offset(codes, codes_off)
    absmax = (torch.rand(cdiv(n, bs), generator=g) * 4 + 1e-3).cuda()
    return codes, absmax


def build_dequantize(dtype, qt, n, bs, seed, codes_off=0, out_off=0):
    codes, absmax = _dequantize_inputs(n, bs, qt, seed, codes_off)
    code = _code() if qt is None else None
    inputs = dict(codes=codes, absmax=absmax, code=code)
    return inputs, lambda: dequantize_guarded(nat.lib, codes, absmax, bs, n, qt, dtype, code, out_off)


def _nested_weight(N, K, qt, dtype, bs, seed):
    import bitsandbytes_b200.functional as F

    g = torch.Generator(device="cpu").manual_seed(seed)
    W = torch.randn(N, K, generator=g).to(nat.DTYPE[dtype]).cuda()
    qW, qs = F.quantize_4bit(W, blocksize=bs, quant_type=qt, compress_statistics=True)
    del W
    return qW, qs


def build_panel(dtype, qt, bs, N, K, n0, rows, seed):
    """Rows [n0, n0 + rows) of an [N, K] weight quantised with nested statistics, through the panel entry."""
    qW, qs = _nested_weight(N, K, qt, dtype, bs, seed)
    off = qs.offset.to(torch.float32).reshape(1).contiguous()

    def go():
        out = torch.full((rows * K + GUARD,), float("nan"), device="cuda", dtype=nat.DTYPE[dtype])
        rc = nat.lib.cbnb_b200_dequantize_4bit_panel(
            qW.data_ptr(), qs.state2.absmax.data_ptr(), qs.absmax.data_ptr(), qs.state2.code.data_ptr(),
            off.data_ptr(), out.data_ptr(), bs, nat.QT_ID[qt], nat.DTYPE_ID[dtype], n0, rows, K, nat.stream())
        sync()
        nat.check()
        assert rc == 0
        return out

    return dict(qW=qW, qs=qs), go


BUILDERS = {"quantize": build_quantize, "dequantize": build_dequantize, "panel": build_panel}


def build(case):
    kind, kwargs = case
    return BUILDERS[kind](**kwargs)


# ----------------------------------------------------------------------- the launch record (profiled children)
_KERNEL = r"\b((?:de)?quantize(?:_blockwise(?:_generic)?|4_prmt)_kernel)<([^<>]*)>"


def _instance(name: str):
    import re

    m = re.search(_KERNEL, name)
    return [m.group(1)] + [_arg(a) for a in m.group(2).split(",")] if m else None


def _profiled(fn):
    """[(demangled name, grid x or None)] of the CUDA kernels of one torch.profiler session around fn(), in launch
    order, read from the session's chrome trace (whose kernel events carry the grid)."""
    from torch.profiler import ProfilerActivity, profile

    sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)  # (the first kernels of a session can go unrecorded)
        sync()
        fn()
        sync()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    kernels = [e for e in events if str(e.get("cat", "")).lower() == "kernel"]
    kernels.sort(key=lambda e: e.get("ts", 0))
    out = []
    for e in kernels:
        grid = e.get("args", {}).get("grid")
        out.append((e.get("name", ""), grid[0] if isinstance(grid, list) and grid else None))
    return out


def record_launches_main():
    """The child: reads a JSON list of cases on stdin and prints one line "LAUNCHES <json>" mapping each case's key to
    {"kernels": [[kernel, template arguments..., grid x]] (None: nothing recorded; a string: the error),
     "digest": SHA-256 of the launches' outputs}, plus "peak_bytes" (the child's peak device allocation)."""
    cases = json.loads(sys.stdin.read())
    for _ in range(5):  # the first sessions of a process can record nothing while the profiler starts up
        if _profiled(lambda: torch.ones(1, device="cuda").mul_(2)):
            break
    record = {}
    for case in cases:
        entry = {"kernels": None, "digest": None}
        try:
            _, go = build(case)
            outs = []
            for _ in range(2):
                kernels = _profiled(lambda: outs.append(go()))
                if kernels:
                    entry["kernels"] = [_instance(name) + [grid] for name, grid in kernels if _instance(name)]
                    break
            o = outs[-1]
            entry["digest"] = digest(o if isinstance(o, tuple) else (o,))
        except Exception as e:  # reported by the test of this case
            entry["kernels"] = f"{type(e).__name__}: {e}"
        record[case_key(case)] = entry
        outs = go = None
        torch.cuda.empty_cache()
    record["peak_bytes"] = torch.cuda.max_memory_allocated()
    print("LAUNCHES " + json.dumps(record), flush=True)


def case_key(case) -> str:
    return json.dumps(case, sort_keys=True)


def _run_child(cases, env=None):
    code = (f"import sys; sys.path.insert(0, {str(ROOT)!r}); "
            "from tests.test_gpu_blockwise_instances import record_launches_main; record_launches_main()")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], input=json.dumps(cases), capture_output=True, text=True,
                       cwd=str(ROOT), timeout=1500, env=env)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("LAUNCHES ")]
    if r.returncode != 0 or not lines:
        pytest.fail(f"the profiled child exited with {r.returncode}:\n{r.stderr[-4000:]}")
    return json.loads(lines[-1][len("LAUNCHES "):])


@pytest.fixture(scope="module")
def launches():
    """{case key: what its launches ran}, recorded once for every test of this file by the profiled child."""
    return _run_child(all_cases())


@pytest.fixture(scope="module")
def walk_launches():
    """The same for the 8-bit quantize cases, in a child whose 8-bit quantizer takes the 7-step code walk."""
    env = dict(os.environ, BNB_B200_Q8_WALK="1")
    return _run_child(walk_cases(), env=env)


NO_RECORD = "torch.profiler recorded no CUDA kernels here: which kernel instance ran is not confirmed"


def recorded(launches, case, want):
    """Asserts the case's launches: `want` is [(instance tuple, grid x)]; the grids are compared when the trace has
    them.  Returns NO_RECORD without a record (the caller skips at its end, after the reference comparison), else
    None."""
    got = launches[case_key(case)]["kernels"]
    if got is None:
        return NO_RECORD
    assert not isinstance(got, str), f"the profiled replay of this case failed: {got}"
    assert [tuple(k[:-1]) for k in got] == [w[0] for w in want], got
    grids = [k[-1] for k in got]
    if all(g is not None for g in grids):
        assert grids == [w[1] for w in want], (grids, want)
    return None


def finish(note):
    if note:
        pytest.skip(note)


def inst(kernel, dtype, *args):
    return (kernel, T_NAME[dtype], *[str(a) for a in args])


# ---------------------------------------------------------------------------------- 2. quantize, every instance
# (dtype, qt, blocksize): every T x {8-bit, NF4, FP4}; blocksizes 32 (G = 2), 64, 256, 1024 (G = 64: the swarp path)
# and 4096 (G = 256)
FAST_ROWS = [
    ("fp32", None, 4096), ("fp16", None, 1024), ("bf16", None, 256), ("fp32", None, 64),
    ("fp32", "nf4", 32), ("fp16", "nf4", 64), ("bf16", "nf4", 4096),
    ("fp32", "fp4", 1024), ("fp16", "fp4", 256), ("bf16", "fp4", 32),
]
FAST_TAIL = 1001  # odd, and not a multiple of 4096: the generic kernel takes the ragged tail


def fast_n():
    """2 full rounds of the fast quantizer plus a partial one (8 S + 8 S + 4 S + 1 tiles), plus the tail."""
    return (20 * sms() + 1) * Q_TILE + FAST_TAIL


def fast_case(dtype, qt, bs):
    return ["quantize", dict(dtype=dtype, qt=qt, n=fast_n(), bs=bs)]


ZERO_CODE = {"nf4": 7, "fp4": 0}


def check_quantize(case, inputs, codes, absmax):
    """Guards, absmax bit for bit and codes within the threshold allowance against the oracle, the padding nibble."""
    kw = case[1]
    qt, n, bs = kw["qt"], kw["n"], kw["bs"]
    assert_quantize_guards(codes, absmax, n, bs, qt)
    nbytes = n if qt is None else (n + 1) // 2
    code = inputs["code"]
    got_q = codes[:nbytes].cpu().numpy()
    _check_codes_vs_oracle(inputs["A"].float().cpu().numpy(), got_q, absmax[:cdiv(n, bs)].cpu().numpy(), bs, qt,
                           None if code is None else code.cpu().numpy())
    if qt is not None and n % 2:
        assert got_q[-1] & 15 == ZERO_CODE[qt], "the padding nibble is not the code of 0.0"


def check_quantize_ref(case, inputs, codes, absmax):
    """Bit for bit against the reference CUDA library (skips the rest of the test when it is not built)."""
    kw = case[1]
    dtype, qt, n, bs = kw["dtype"], kw["qt"], kw["n"], kw["bs"]
    nbytes, nb = (n if qt is None else (n + 1) // 2), cdiv(n, bs)
    ref = nat.ref_cuda()
    rq, rabs = quantize_guarded(ref, inputs["A"], bs, qt, dtype, inputs["code"])
    assert torch.equal(f_view(rabs[:nb]), f_view(absmax[:nb])), "absmax differs from the reference"
    neq = (rq[:nbytes] != codes[:nbytes]).sum().item()
    assert neq == 0, f"{neq} codes differ from the reference CUDA kernel"


def f_view(t):
    return t.view(torch.int32)


@pytest.mark.parametrize("dtype,qt,bs", FAST_ROWS)
def test_quantize_fast_path_rounds(launches, dtype, qt, bs):
    """quantize_blockwise_kernel<T, QT> over 3 grid-stride rounds (the last one partial), then
    quantize_blockwise_generic_kernel<T, QT> on the ragged tail; n odd, so the last byte's low nibble is padding."""
    case = fast_case(dtype, qt, bs)
    n = case[1]["n"]
    inputs, go = build(case)
    codes, absmax = go()
    nat.check()
    tiles = n // Q_TILE
    grid = capped(tiles, Q_CAP)
    assert rounds(tiles, grid, 1) == 3
    tail_blocks = cdiv(n, bs) - tiles * Q_TILE // bs
    want = [(inst("quantize_blockwise_kernel", dtype, QT_ARG[qt]), grid),
            (inst("quantize_blockwise_generic_kernel", dtype, QT_ARG[qt]), capped(cdiv(tail_blocks, QG_WARPS), QG_CAP))]
    check_quantize(case, inputs, codes, absmax)
    note = recorded(launches, case, want)
    check_quantize_ref(case, inputs, codes, absmax)
    finish(note)


# 8-bit cases of the walk child: multi-round fast bodies plus tails, every T
WALK_ROWS = [("fp32", None, 4096), ("fp16", None, 1024), ("bf16", None, 256), ("fp32", None, 64)]


@pytest.mark.parametrize("dtype,qt,bs", WALK_ROWS)
def test_quantize_walk_equals_bracket_search(walk_launches, dtype, qt, bs):
    """BNB_B200_Q8_WALK=1: quantize_blockwise_kernel<T, 0> and quantize_blockwise_generic_kernel<T, 0> (the reference's
    7-step walk) write the same bytes, guards included, as the default bracket search in this process."""
    case = fast_case(dtype, qt, bs)
    _, go = build(case)
    codes, absmax = go()
    nat.check()
    entry = walk_launches[case_key(case)]
    assert not isinstance(entry["kernels"], str), entry["kernels"]
    assert entry["digest"] == digest((codes, absmax)), "the 7-step walk and the bracket search differ"
    n = case[1]["n"]
    tiles = n // Q_TILE
    tail_blocks = cdiv(n, bs) - tiles * Q_TILE // bs
    finish(recorded(walk_launches, case, [(inst("quantize_blockwise_kernel", dtype, 0), capped(tiles, Q_CAP)),
                                          (inst("quantize_blockwise_generic_kernel", dtype, 0),
                                           capped(cdiv(tail_blocks, QG_WARPS), QG_CAP))]))


# (dtype, qt, blocksize, activation offset in elements, quant blocks in units of 64 S): the generic kernel alone,
# over more than one round of 64 S blocks
GENERIC_ROWS = [
    pytest.param("bf16", None, 64, 1, 3.5, id="A+1-bf16-8bit-bs64"),
    pytest.param("fp32", "nf4", 128, 1, 2.5, id="A+1-fp32-nf4-bs128"),
    pytest.param("fp16", "fp4", 32, 1, 3.5, id="A+1-fp16-fp4-bs32"),
    pytest.param("fp32", None, 48, 0, 2.5, id="bs48-fp32-8bit"),
    pytest.param("bf16", "nf4", 48, 0, 3.5, id="bs48-bf16-nf4"),
    pytest.param("fp16", "fp4", 8192, 0, 1.1, id="bs8192-fp16-fp4"),
]


def generic_case(dtype, qt, bs, a_off, blocks):
    nblocks = int(blocks * 64 * sms())
    return ["quantize", dict(dtype=dtype, qt=qt, n=(nblocks - 1) * bs + 37, bs=bs, a_off=a_off)]


@pytest.mark.parametrize("dtype,qt,bs,a_off,blocks", GENERIC_ROWS)
def test_quantize_generic_routes(launches, dtype, qt, bs, a_off, blocks):
    """quantize_blockwise_generic_kernel<T, QT> alone: activations 1 element past a 16-byte boundary, an even
    non-power-of-two blocksize (48: the oracle only, the reference does not serve it) and a blocksize above 4096,
    each over more than 64 S quant blocks (the kernel loops), the last block ragged."""
    case = generic_case(dtype, qt, bs, a_off, blocks)
    n = case[1]["n"]
    inputs, go = build(case)
    codes, absmax = go()
    nat.check()
    nblocks = cdiv(n, bs)
    grid = capped(cdiv(nblocks, QG_WARPS), QG_CAP)
    assert rounds(nblocks, grid, QG_WARPS) >= 2
    check_quantize(case, inputs, codes, absmax)
    note = recorded(launches, case, [(inst("quantize_blockwise_generic_kernel", dtype, QT_ARG[qt]), grid)])
    if bs & (bs - 1) == 0 and bs <= 4096 and (qt is not None or bs >= 64):
        check_quantize_ref(case, inputs, codes, absmax)
    finish(note)


# ------------------------------------------------------------------------------- 3. dequantize, every instance
def dq_round(dtype):
    """Elements one round of dequantize_blockwise_kernel writes: 8 S x 2048 vectors of 16 bytes."""
    return DQ_CAP * sms() * DQ_VECS * (16 // torch.tensor([], dtype=nat.DTYPE[dtype]).element_size())


def d4_round():
    return D4_CAP * sms() * D4_UNITS * 64


# (name, dtype, qt, blocksize, rounds of the persistent kernel, extra elements, codes offset, the persistent kernel)
DEQ_ROWS = [
    pytest.param("fp32", None, 256, 3.5, 3, 0, "vec", id="8bit-fp32-bs256"),
    pytest.param("fp16", None, 4096, 3.5, 5, 0, "vec", id="8bit-fp16-bs4096"),
    pytest.param("bf16", None, 64, 3.5, 7, 0, "vec", id="8bit-bf16-bs64"),
    pytest.param("fp32", "nf4", 64, 3.5, 1, 0, "vec", id="nf4-fp32-bs64"),
    pytest.param("fp32", "fp4", 1024, 3.5, 2, 0, "vec", id="fp4-fp32-bs1024"),
    pytest.param("fp16", "nf4", 128, 3.5, 9, 8, "vec", id="nf4-fp16-codes+8"),
    pytest.param("bf16", "fp4", 16, 3.5, 3, 0, "vec", id="fp4-bf16-bs16"),
    pytest.param("bf16", "nf4", 256, 0.3, 5, 8, "vec", id="nf4-bf16-codes+8"),
    pytest.param("fp16", "fp4", 16, 0.3, 0, 0, "vec", id="fp4-fp16-bs16"),
    pytest.param("bf16", "nf4", 64, 3.5, 37, 0, "prmt", id="prmt-nf4-bf16-bs64-tail37"),
    pytest.param("fp16", "fp4", 32, 3.5, 0, 0, "prmt", id="prmt-fp4-fp16-bs32"),
    pytest.param("bf16", "fp4", 32, 3.5, 37, 0, "prmt", id="prmt-fp4-bf16-bs32-tail37"),
    pytest.param("fp16", "nf4", 4096, 1.5, 0, 0, "prmt", id="prmt-nf4-fp16-bs4096"),
]


def deq_case(dtype, qt, bs, nrounds, extra, codes_off, kernel):
    per_round = d4_round() if kernel == "prmt" else dq_round(dtype)
    n = int(nrounds * per_round) // 64 * 64 + extra
    return ["dequantize", dict(dtype=dtype, qt=qt, n=n, bs=bs, seed=n % 9973 + bs, codes_off=codes_off)]


def check_dequantize(case, inputs, buf):
    kw = case[1]
    dtype, qt, n, bs, out_off = kw["dtype"], kw["qt"], kw["n"], kw["bs"], kw.get("out_off", 0)
    assert_dequantize_guards(buf, n, out_off)
    codes, absmax, code = inputs["codes"], inputs["absmax"], inputs["code"]
    want = oracle.dequantize_blockwise(codes.cpu().numpy(), absmax.cpu().numpy(), bs, n, qt,
                                       None if code is None else code.cpu().numpy(), dtype)
    check_dequantized(out_bits(buf[out_off:out_off + n]), want.view(np.uint32) if dtype == "fp32" else want, dtype)


def check_dequantize_ref(case, inputs, buf):
    """Bit for bit against the reference CUDA library where it serves the case (power-of-two blocksizes, 8-bit from
    64, 4-bit from 32); skips the rest of the test when it is not built."""
    kw = case[1]
    dtype, qt, n, bs, out_off = kw["dtype"], kw["qt"], kw["n"], kw["bs"], kw.get("out_off", 0)
    if bs & (bs - 1) != 0 or bs < (64 if qt is None else 32):
        return
    ref = nat.ref_cuda()
    rbuf = dequantize_guarded(ref, inputs["codes"], inputs["absmax"], bs, n, qt, dtype, inputs["code"], out_off)
    assert np.array_equal(out_bits(rbuf[out_off:out_off + n]), out_bits(buf[out_off:out_off + n])), \
        "differs from the reference"


@pytest.mark.parametrize("dtype,qt,bs,nrounds,extra,codes_off,kernel", DEQ_ROWS)
def test_dequantize_rounds(launches, dtype, qt, bs, nrounds, extra, codes_off, kernel):
    """The persistent dequantizers over several grid-stride rounds (the last partial), the generic kernel on the tail:
    dequantize_blockwise_kernel<T, 0> for every T, <float, FP4 | NF4>, and <T16, FP4 | NF4> for codes 8 bytes past a
    16-byte boundary or blocksize 16; dequantize4_prmt_kernel<T16, QT, false> with blocksize 32 (two tables per unit)
    and n = 64 k + 37 (the <<<1, 256>>> tail launch)."""
    case = deq_case(dtype, qt, bs, nrounds, extra, codes_off, kernel)
    n = case[1]["n"]
    inputs, go = build(case)
    buf = go()
    nat.check()
    T = T_NAME[dtype]
    if kernel == "prmt":
        units = n // 64
        grid = capped(cdiv(units, D4_UNITS), D4_CAP)
        nr = rounds(units, grid, D4_UNITS)
        want = [(("dequantize4_prmt_kernel", T, DQ_QT_ARG[qt], "0"), grid)]
        first = units * 64
        tail_grid = 1
    else:
        oe = 16 // buf.element_size()
        n_vec = n // oe
        grid = capped(cdiv(n_vec, DQ_VECS), DQ_CAP)
        nr = rounds(n_vec, grid, DQ_VECS)
        want = [(("dequantize_blockwise_kernel", T, DQ_QT_ARG[qt]), grid)]
        first = n_vec * oe
        tail_grid = capped(cdiv(n - first, DG_ELEMS), DG_CAP)
    assert nr == int(np.ceil(nrounds)), nr
    if first < n:
        want.append((("dequantize_blockwise_generic_kernel", T, DQ_QT_ARG[qt]), tail_grid))
    check_dequantize(case, inputs, buf)
    note = recorded(launches, case, want)
    check_dequantize_ref(case, inputs, buf)
    finish(note)


# (dtype, qt, blocksize, output offset in elements): dequantize_blockwise_generic_kernel alone, over 4 rounds
DEQ_GENERIC_ROWS = [
    pytest.param("bf16", "nf4", 64, 1, id="out+1-bf16-nf4"),
    pytest.param("fp16", None, 256, 1, id="out+1-fp16-8bit"),
    pytest.param("fp32", "fp4", 128, 1, id="out+1-fp32-fp4"),
    pytest.param("fp16", None, 48, 0, id="bs48-fp16-8bit"),
    pytest.param("fp32", "nf4", 48, 0, id="bs48-fp32-nf4"),
    pytest.param("bf16", "fp4", 33, 0, id="bs33-bf16-fp4"),
]


def deq_generic_case(dtype, qt, bs, out_off):
    n = int(3.5 * DG_CAP * sms() * DG_ELEMS) + 7
    return ["dequantize", dict(dtype=dtype, qt=qt, n=n, bs=bs, seed=bs + out_off, out_off=out_off)]


@pytest.mark.parametrize("dtype,qt,bs,out_off", DEQ_GENERIC_ROWS)
def test_dequantize_generic_routes(launches, dtype, qt, bs, out_off):
    """dequantize_blockwise_generic_kernel<T, QT> alone, over 4 grid-stride rounds: an output 1 element (2 or 4 bytes)
    off alignment, non-power-of-two blocksizes (48, and 33 for 4-bit codes: decoding needs no even blocksize)."""
    case = deq_generic_case(dtype, qt, bs, out_off)
    n = case[1]["n"]
    inputs, go = build(case)
    buf = go()
    nat.check()
    grid = capped(cdiv(n, DG_ELEMS), DG_CAP)
    assert rounds(n, grid, DG_ELEMS) == 4
    check_dequantize(case, inputs, buf)
    note = recorded(launches, case, [(inst("dequantize_blockwise_generic_kernel", dtype, DQ_QT_ARG[qt]), grid)])
    check_dequantize_ref(case, inputs, buf)
    finish(note)


# ------------------------------------------------------------------ 4. the nested-statistics decoders at scale
def pin_nested_dequantize_4bit(qW, qs, dtype, want):
    """F.dequantize_4bit with nested statistics == the oracle's decode with oracle.nested_absmax, bit for bit."""
    a = oracle.nested_absmax(qs.state2.absmax.cpu().numpy(), qs.absmax.cpu().numpy(), qs.state2.code.cpu().numpy(),
                             float(qs.offset.item()))
    n = want.numel()
    w = oracle.dequantize_blockwise(qW.cpu().numpy().reshape(-1), a, qs.blocksize, n, qs.quant_type, None, dtype)
    check_dequantized(nat.to_bits(want.reshape(-1)), w, "F.dequantize_4bit")


# (dtype, qt, blocksize, K, n0, rounds): K = 4160 is not a multiple of the blocksize 4096
PANEL_ROWS = [
    pytest.param("bf16", "nf4", 4096, 4160, 256, 3.5, id="bf16-nf4-bs4096-K4160"),
    pytest.param("fp16", "fp4", 4096, 4160, 384, 3.5, id="fp16-fp4-bs4096-K4160"),
    pytest.param("bf16", "fp4", 32, 1024, 128, 1.5, id="bf16-fp4-bs32"),
    pytest.param("fp16", "nf4", 32, 1024, 128, 1.5, id="fp16-nf4-bs32"),
]


def panel_case(dtype, qt, bs, K, n0, nrounds):
    rows = cdiv(int(nrounds * d4_round()), K)
    return ["panel", dict(dtype=dtype, qt=qt, bs=bs, N=n0 + rows + 128, K=K, n0=n0, rows=rows, seed=K + n0)]


@pytest.mark.parametrize("dtype,qt,bs,K,n0,nrounds", PANEL_ROWS)
def test_nested_panel_decode(launches, dtype, qt, bs, K, n0, nrounds):
    """dequantize4_prmt_kernel<T16, QT, true> through cbnb_b200_dequantize_4bit_panel at a non-zero row offset, over
    up to 4 grid-stride rounds: the same bits as the same rows of F.dequantize_4bit (compress_statistics=True), which
    is itself pinned to the oracle's decode with oracle.nested_absmax."""
    import bitsandbytes_b200.functional as F

    case = panel_case(dtype, qt, bs, K, n0, nrounds)
    rows, N = case[1]["rows"], case[1]["N"]
    inputs, go = build(case)
    buf = go()
    assert (out_bits(buf[rows * K:]) == out_bits(torch.full((1,), float("nan"), dtype=buf.dtype))[0]).all()
    units = rows * K // 64
    grid = capped(cdiv(units, D4_UNITS), D4_CAP)
    assert rounds(units, grid, D4_UNITS) == int(np.ceil(nrounds))
    qW, qs = inputs["qW"], inputs["qs"]
    want = F.dequantize_4bit(qW, qs).view(N, K)
    got = buf[:rows * K].view(rows, K)
    check_dequantized(nat.to_bits(got).reshape(-1), nat.to_bits(want[n0:n0 + rows]).reshape(-1), "panel")
    pin_nested_dequantize_4bit(qW, qs, dtype, want)
    finish(recorded(launches, case, [(("dequantize4_prmt_kernel", T_NAME[dtype], DQ_QT_ARG[qt], "1"), grid)]))


# ------------------------------------------------------------------------ 5. edges where fast-math kernels go wrong
FLT_MIN = np.float32(2.0**-126)
EDGE_BS = 64


def _edge_blocks(dtype, qt):
    """Nine blocks of 64 elements, one edge each (named in the returned list)."""
    g = np.random.default_rng(5)
    blocks = []

    def normal():
        return g.standard_normal(EDGE_BS).astype(np.float32)

    b = normal()
    b[::7] = np.float32(2.0**-130) * np.sign(b[::7])  # subnormal values (bf16 has them too) in a normal block
    blocks.append(("subnormals-in-a-normal-block", b))
    blocks.append(("all-subnormal", (g.standard_normal(EDGE_BS) * 2.0**-130).astype(np.float32)))
    b = (normal() * 2.0**-121).astype(np.float32)
    b[0] = 1024.0  # x * rcp(1024) < 2^-126 for every other element
    blocks.append(("products-underflow", b))
    b = normal()
    b[5] = np.float32(2.0**126) * 1.5
    blocks.append(("max-at-least-2^126", b))
    b = normal()
    b[9], b[40] = np.inf, -np.inf
    blocks.append(("plus-minus-inf", b))
    b = normal()
    b[17] = np.nan
    blocks.append(("one-nan", b))
    blocks.append(("all-nan", np.full(EDGE_BS, np.nan, np.float32)))
    if qt is None:
        cb = _code().cpu().numpy()
        mids = (cb[:-1] + cb[1:]) * np.float32(0.5)
    else:
        lut = oracle.lut4(qt)
        s = np.sort(lut)
        mids = (s[:-1] + s[1:]) * np.float32(0.5)
    b = np.resize(mids, EDGE_BS).astype(np.float32)
    b[0] = 1.0  # absmax 1: x * rcp(1) is the midpoint itself
    blocks.append(("code-book-midpoints", b))
    b = np.resize(mids, EDGE_BS).astype(np.float32) * np.float32(4.0)
    b[0] = -4.0
    blocks.append(("midpoints-times-4", b))
    names = [nm for nm, _ in blocks]
    A = np.concatenate([b for _, b in blocks])
    return names, A


def _ftz(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, np.float32)
    return np.where(np.abs(x) < FLT_MIN, np.copysign(np.float32(0), x), x).astype(np.float32)


EDGE_DTYPES = ["fp32", "bf16"]
EDGE_QTS = [None, "nf4", "fp4"]


@pytest.mark.parametrize("qt", EDGE_QTS, ids=["8bit", "nf4", "fp4"])
@pytest.mark.parametrize("dtype", EDGE_DTYPES)
def test_quantize_edges(dtype, qt):
    """Subnormals, underflowing products, |x| >= 2^126, +-inf, NaN, all-NaN and code-book midpoints, one block each:
    absmax is the maximum of the flushed |x| with NaN ignored (-FLT_MAX for an all-NaN block); with the reference
    built, codes and absmax equal the reference CUDA kernel's bit for bit."""
    names, A32 = _edge_blocks(dtype, qt)
    if dtype == "fp32":
        A = torch.from_numpy(A32).cuda()
    else:
        A = torch.from_numpy(A32).to(torch.bfloat16).cuda()
        A32 = A.float().cpu().numpy()
    code = _code() if qt is None else None
    n = A.numel()
    codes, absmax = quantize_guarded(nat.lib, A, EDGE_BS, qt, dtype, code)
    nat.check()
    assert_quantize_guards(codes, absmax, n, EDGE_BS, qt)
    mag = np.abs(_ftz(A32)).reshape(-1, EDGE_BS)
    want = np.where(np.isnan(mag), np.float32(-3.4028234663852886e38), mag).max(axis=1).astype(np.float32)
    got = absmax[:n // EDGE_BS].cpu().numpy()
    for i, nm in enumerate(names):
        assert got[i].view(np.uint32) == want[i].view(np.uint32), (nm, got[i], want[i])
    ref = nat.ref_cuda()
    rq, rabs = quantize_guarded(ref, A, EDGE_BS, qt, dtype, code)
    nbytes = n if qt is None else n // 2
    assert torch.equal(f_view(rabs[:n // EDGE_BS]), f_view(absmax[:n // EDGE_BS]))
    per = EDGE_BS if qt is None else EDGE_BS // 2
    for i, nm in enumerate(names):
        sl = slice(i * per, (i + 1) * per)
        assert torch.equal(rq[:nbytes][sl], codes[:nbytes][sl]), (nm, codes[sl].tolist(), rq[sl].tolist())


def _dequantize_edge_expectation(values, scale, dtype):
    """rn_T(value * absmax) under FTZ: a subnormal absmax reads as a zero of its sign, a subnormal product is flushed
    to a zero of the product's sign, then one rounding to T."""
    with np.errstate(all="ignore"):
        p = (values.astype(np.float32) * _ftz(scale)).astype(np.float32)
        return oracle.round_to(_ftz(p), dtype)


# absmax per 64-element block: normal, products underflowing (some), subnormal (two), 2^127, inf, NaN
EDGE_ABSMAX = np.array([1.5, 2.0**-120, 2.0**-127 * 1.5, 2.0**-149, 2.0**127, np.inf, np.nan, 3.0], np.float32)


@pytest.mark.parametrize("qt", EDGE_QTS, ids=["8bit", "nf4", "fp4"])
@pytest.mark.parametrize("dtype", EDGE_DTYPES)
@pytest.mark.parametrize("out_off", [0, 1], ids=["aligned", "out+1"])
def test_dequantize_edges(dtype, qt, out_off):
    """Every code value times a normal, an underflowing, a subnormal, a huge, an infinite and a NaN absmax: the FTZ
    expectation (_dequantize_edge_expectation) bit for bit, NaN where it is NaN, with or without the reference.  The
    aligned output takes the persistent kernels (dequantize_blockwise_kernel, or dequantize4_prmt_kernel for 4-bit into
    bf16), the offset one the generic kernel."""
    nb = EDGE_ABSMAX.size
    n = nb * EDGE_BS
    e = np.arange(n)
    if qt is None:
        codes_np = ((e * 37 + e // EDGE_BS) % 256).astype(np.uint8)
        values = _code().cpu().numpy()[codes_np]
    else:
        nib = ((e * 5 + e // EDGE_BS) % 16).astype(np.uint8)
        codes_np = ((nib[0::2] << 4) | nib[1::2]).astype(np.uint8)
        values = oracle.lut4(qt)[nib]
    scale = EDGE_ABSMAX[e // EDGE_BS]
    want = _dequantize_edge_expectation(values, scale, dtype)
    codes = torch.from_numpy(codes_np).cuda()
    absmax = torch.from_numpy(EDGE_ABSMAX).cuda()
    code = _code() if qt is None else None
    buf = dequantize_guarded(nat.lib, codes, absmax, EDGE_BS, n, qt, dtype, code, out_off)
    nat.check()
    assert_dequantize_guards(buf, n, out_off)
    got = buf[out_off:out_off + n]
    got_f = got.float().cpu().numpy()
    want_f = oracle.widen(want, dtype) if dtype != "fp32" else want
    nan = np.isnan(want_f)
    assert np.array_equal(np.isnan(got_f), nan), np.nonzero(np.isnan(got_f) != nan)[0][:8]
    gb, wb = out_bits(got), (want.view(np.uint32) if dtype == "fp32" else want)
    bad = np.nonzero((gb != wb) & ~nan)[0]
    assert bad.size == 0, [(int(i), int(i) // EDGE_BS, hex(int(gb[i])), hex(int(wb[i]))) for i in bad[:8]]


# ---------------------------------------------------------------------------------- 6. blocksizes that are refused
def _refused(call):
    sync()
    call()
    sync()
    with pytest.raises(RuntimeError, match="blocksize"):
        nat.check()


@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("bs", [33, 63, 1])
def test_odd_blocksize_4bit_quantize_is_refused(dtype, qt, bs):
    """An odd blocksize starts every other block in the middle of a byte: the 4-bit quantize entries (and the
    stream-taking entry) refuse it, set the error message and write nothing."""
    n = 33 * 64 + 1
    A = _inputs(n, dtype)
    codes, absmax = quantize_guarded(nat.lib, A, bs, qt, dtype, None)
    with pytest.raises(RuntimeError, match="blocksize"):
        nat.check()
    assert (codes == SENTINEL_BYTE).all() and (f32_bits(absmax) == SENTINEL_F32).all(), "a refused call wrote"
    out = torch.full((n,), SENTINEL_BYTE, device="cuda", dtype=torch.uint8)
    _refused(lambda: nat.lib.cbnb_b200_quantize_blockwise(None, A.data_ptr(), absmax.data_ptr(), out.data_ptr(), bs, n,
                                                          nat.QT_ID[qt], nat.DTYPE_ID[dtype], nat.stream()))
    assert (out == SENTINEL_BYTE).all()


@pytest.mark.parametrize("qt", [None, "nf4", "fp4"], ids=["8bit", "nf4", "fp4"])
@pytest.mark.parametrize("bs", [0, -64])
def test_blocksize_below_one_is_refused(qt, bs):
    """Blocksize < 1 divides by zero (or indexes backwards): every quantize and dequantize entry refuses it with the
    error message set and writes nothing."""
    n = 1000
    code = _code() if qt is None else None
    for dtype in ("fp32", "fp16", "bf16"):
        A = _inputs(n, dtype)
        codes = torch.full((n + GUARD,), SENTINEL_BYTE, device="cuda", dtype=torch.uint8)
        absmax = torch.full((GUARD,), 1.0, device="cuda")
        fn = getattr(nat.lib, f"cquantize_blockwise_{dtype}" + ("" if qt is None else f"_{qt}"))
        _refused(lambda: fn(nat.ptr(code), A.data_ptr(), absmax.data_ptr(), codes.data_ptr(), bs, n))
        _refused(lambda: nat.lib.cbnb_b200_quantize_blockwise(nat.ptr(code), A.data_ptr(), absmax.data_ptr(),
                                                              codes.data_ptr(), bs, n, nat.QT_ID[qt],
                                                              nat.DTYPE_ID[dtype], nat.stream()))
        assert (codes == SENTINEL_BYTE).all() and (absmax == 1.0).all(), dtype
        buf = torch.full((n,), float("nan"), device="cuda", dtype=nat.DTYPE[dtype])
        dq = getattr(nat.lib, f"cdequantize_blockwise_{dtype}" + ("" if qt is None else f"_{qt}"))
        _refused(lambda: dq(nat.ptr(code), codes.data_ptr(), absmax.data_ptr(), buf.data_ptr(), bs, n, nat.stream()))
        assert torch.isnan(buf.float()).all(), dtype


# ------------------------------------------------------------------------------------- every case of the file
def walk_cases():
    return [fast_case(*r) for r in WALK_ROWS]


def all_cases():
    """The case of every test above that records its launches, in the order the child replays them."""
    cases = [fast_case(*r) for r in FAST_ROWS]
    cases += [generic_case(*r.values) for r in GENERIC_ROWS]
    cases += [deq_case(*r.values) for r in DEQ_ROWS]
    cases += [deq_generic_case(*r.values) for r in DEQ_GENERIC_ROWS]
    cases += [panel_case(*r.values) for r in PANEL_ROWS]
    return cases
