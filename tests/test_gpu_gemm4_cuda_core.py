"""GPU parity: the 4-bit GEMM's decode-regime and CUDA-core kernels, every instance, against the float64 oracle.

Three kernels serve every 4-bit GEMM that the wgmma GEMM does not:

* ``gemv4_fast_kernel<T, QT, MB, PART>`` (gemv4_simt.cu): <= 8 tokens of 16-bit activations, K % 32 == 0, a
  power-of-two blocksize >= 32, 16-byte aligned operands.  MB = 1, 2, 4 or 8 token slots.
* ``gemv4_simt_kernel<T, PART, VEC>`` (gemv4_simt.cu): everything else -- every fp32 call at default precision, any
  K % 64 != 0 beyond the fast kernel, misaligned operands, any blocksize.  VEC = the vector body (K % 8 == 0,
  blocksize % 8 == 0, 16-byte aligned activations, 4-byte aligned codes), otherwise the scalar body.
* ``gemv4_mma_kernel<T, QT, W, NT, PART>`` (gemv4_mma.cu): the mma.sync decode kernel, up to 16 tokens.  W = 4, 8
  or 16 warps per CTA (by the row-tile count and K), NT = 1 or 2 groups of 8 tokens.

Every call goes through the C ABI (plain, strided, partial and scatter entries, the legacy GEMV entry), into an
output filled with NaN so that an unwritten element fails.  The bound is the suite's: half an ulp of T plus the fp32
accumulation term (test_gpu_gemm4.assert_close_to_exact) for T outputs, and the fp32 partial bound of
test_gpu_row_parallel for the partial entries.

Which instance ran is proven from the kernel names: one child process (the same interpreter, which exits when done)
replays every test's launches under torch.profiler and reports the demangled name and template arguments of each
4-bit GEMM kernel it launched, and each test asserts on its own list.  The child keeps the profiler out of the pytest
process, where a session changes what later profiler sessions of other tests record.  Each test's launches are the
same function call in both processes (the launch_* functions below take only JSON arguments and seeded inputs).
"""
import ctypes as ct
import json
import re
import subprocess
import sys
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from tests import _native as nat
from tests.test_gpu_gemm4 import assert_close_to_exact, exact, make_problem, run
from tests.test_gpu_gemm4_tf32 import accumulation, precision, ulp32  # noqa: F401

pytestmark = pytest.mark.gpu

SIMT_MAX_TOKEN_GROUPS = 65535  # gridDim.y limit: the CUDA-core kernel's 4-token groups per launch
ROOT = Path(__file__).resolve().parent.parent
T_NAME = {"bf16": "__nv_bfloat16", "fp16": "__half", "fp32": "float"}  # T as the demangled kernel name spells it
QT_ARG = {"fp4": "1", "nf4": "2"}  # QuantType kFP4 / kNF4
QTS = ["nf4", "fp4"]
DT16 = ["bf16", "fp16"]


@contextmanager
def forced(path):
    """Forces the 4-bit GEMM's kernel choice for the calls inside (None: the dispatcher's own choice)."""
    if path is None:
        yield
        return
    nat.lib.cbnb_b200_gemm_4bit_force_path(path)
    try:
        yield
    finally:
        nat.lib.cbnb_b200_gemm_4bit_force_path(-1)


def make_problem_any_bs(M, N, K, qt, dtype, bs, nested=False, bias=False, seed=0):
    """make_problem for any blocksize: a power of two as the library quantises, otherwise (the C entries take any
    blocksize; the Python layer refuses it) codes and absmax from the oracle's quantize_blockwise."""
    if bs & (bs - 1) == 0:
        return make_problem(M, N, K, qt, dtype, bs=bs, nested=nested, bias=bias, seed=seed)
    g = torch.Generator(device="cpu").manual_seed(seed * 7919 + M * 31 + N * 17 + K)
    W = (torch.randn(N, K, generator=g) / K**0.5).to(nat.DTYPE[dtype])
    x = torch.randn(M, K, generator=g).to(nat.DTYPE[dtype]).cuda()
    codes, absmax = oracle.quantize_blockwise(oracle.widen(nat.to_bits(W).reshape(-1), dtype), bs, qt)
    p = dict(x=x, packed=torch.from_numpy(codes).cuda(), absmax=torch.from_numpy(absmax).cuda(), M=M, N=N, K=K, bs=bs,
             qt=qt, dtype=dtype, bias=None, absmax_8bit=None, absmax_code=None, absmax_offset=None)
    if nested:
        from bitsandbytes_b200.functional import create_dynamic_map

        code2 = create_dynamic_map().cuda()
        offset = p["absmax"].mean().reshape(1)
        a8, a2 = nat.quantize(nat.lib, (p["absmax"] - offset).contiguous(), 256, None, code2, "fp32")
        p.update(absmax=a2, absmax_8bit=a8, absmax_code=code2, absmax_offset=offset)
    if bias:
        p["bias"] = torch.randn(N, generator=g).to(nat.DTYPE[dtype]).cuda()
    return p


def at_offset(t: torch.Tensor, elems: int) -> torch.Tensor:
    """A contiguous copy of t that starts `elems` elements past an allocation's start (A.contiguous() keeps it)."""
    buf = torch.empty(t.numel() + elems, dtype=t.dtype, device=t.device)
    view = buf[elems:].view(t.shape)
    view.copy_(t)
    assert view.is_contiguous() and view.data_ptr() % 16 == (elems * t.element_size()) % 16
    return view


def strided(p, out, ldc):
    nat.lib.cbnb_b200_gemm_4bit_strided(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
        nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]), out.data_ptr(), nat.ptr(p["bias"]), p["M"], p["N"],
        p["K"], ldc, p["bs"], nat.QT_ID[p["qt"]], nat.DTYPE_ID[p["dtype"]], nat.stream())


def partial(p, outs, ldc):
    ptrs = (ct.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
    rc = nat.lib.cbnb_b200_gemm_4bit_partial(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
        nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]), ct.cast(ptrs, ct.c_void_p), len(outs), p["M"],
        p["N"], p["K"], ldc, p["bs"], nat.QT_ID[p["qt"]], nat.DTYPE_ID[p["dtype"]], nat.stream())
    assert rc == 0


def partial_scatter(p, outs, ldc):
    ptrs = (ct.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
    rc = nat.lib.cbnb_b200_gemm_4bit_partial_scatter(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
        nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]), ct.cast(ptrs, ct.c_void_p), len(outs),
        p["M"] // len(outs), p["M"], p["N"], p["K"], ldc, p["bs"], nat.QT_ID[p["qt"]], nat.DTYPE_ID[p["dtype"]],
        nat.stream())
    assert rc == 0


def assert_partial_close(part: torch.Tensor, y64: np.ndarray, K: int):
    """The fp32 partial against the float64 sum: half an fp32 ulp plus the fp32 accumulation bound
    (test_gpu_row_parallel.test_partial_gemm_vs_float64_oracle)."""
    y = torch.from_numpy(y64).to(part.device)
    assert torch.isfinite(part).all(), "unwritten partial outputs"
    tol = 0.5 * ulp32(y) + accumulation(K, y)
    err = (part.double() - y).abs()
    bad = err > tol
    assert not bad.any(), f"{int(bad.sum())} / {bad.numel()} partials off; worst {float((err / tol).max()):.2f} x tol"


def check_plain_and_partial(p, out, part):
    """The strided output (row stride N + pad) and the partial of launch_routes: the T output meets the oracle bound
    and leaves the columns past N at their fill, the fp32 partial meets the fp32 bound, and T(partial + bias) is the T
    output bit for bit."""
    N, K, dt = p["N"], p["K"], p["dtype"]
    assert torch.isnan(out[:, N:]).all() and torch.isnan(part[:, N:]).all(), "wrote past N"
    got = out[:, :N]
    assert_close_to_exact(got, exact(p), dt, K)
    assert_partial_close(part[:, :N], exact(dict(p, bias=None)), K)
    summed = part[:, :N] + (p["bias"].float() if p["bias"] is not None else 0.0)
    assert torch.equal(summed.to(got.dtype).view(-1).view(torch.uint8), got.contiguous().view(-1).view(torch.uint8))


# ------------------------------------------------------------------------ the launches of each test (seeded inputs)
def launch_routes(dtype, M, N, K, bs, qt, nested, bias, seed, a_off=0, codes_off=0, path=None, pad=3):
    """The strided entry (ldc = N + pad) and the partial entry on one problem, activations `a_off` elements and codes
    `codes_off` bytes past an allocation's start, `path` forced (None: unforced).  Returns (problem, out, partial)."""
    p = make_problem_any_bs(M, N, K, qt, dtype, bs, nested=nested, bias=bias, seed=seed)
    if a_off:
        p["x"] = at_offset(p["x"], a_off)
    if codes_off:
        p["packed"] = at_offset(p["packed"], codes_off)
    ldc = N + pad
    out = torch.full((M, ldc), float("nan"), device="cuda", dtype=nat.DTYPE[dtype])
    part = torch.full((M, ldc), float("nan"), device="cuda", dtype=torch.float32)
    with forced(path):
        strided(p, out, ldc)
        partial(p, [part], ldc)
    torch.cuda.synchronize()
    nat.check()
    return p, out, part


def launch_fallback(dtype, M, N, K, seed):
    """The plain call on activations at a 1-element offset, then on the aligned original."""
    p = make_problem(M, N, K, "nf4", dtype, nested=True, bias=True, seed=seed)
    q = dict(p, x=at_offset(p["x"], 1))
    misaligned = run(nat.lib, q)
    aligned = run(nat.lib, p)
    nat.check()
    return p, misaligned, aligned


def launch_matmul(M, N, K, seed):
    """matmul_4bit on a bf16 activation view at a 1-element offset."""
    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    g = torch.Generator(device="cpu").manual_seed(seed)
    W = (torch.randn(N, K, generator=g) / K**0.5).to(torch.bfloat16).cuda()
    x = at_offset(torch.randn(M, K, generator=g).to(torch.bfloat16).cuda(), 1)
    qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="nf4")
    with torch.no_grad():
        y = bnb.matmul_4bit(x, qW.t(), qs)
    torch.cuda.synchronize()
    return x, qW, qs, y


def launch_plain(dtype, M, N, K, qt, nested, bias, seed):
    p = make_problem(M, N, K, qt, dtype, nested=nested, bias=bias, seed=seed)
    got = run(nat.lib, p)
    nat.check()
    return p, got


def launch_scatter(dtype, M, N, K, qt, nested, seed, parts, pad):
    """The partial scatter entry: M rows over `parts` destinations of M / parts rows (row stride N + pad)."""
    p = make_problem(M, N, K, qt, dtype, nested=nested, seed=seed)
    outs = [torch.full((M // parts, N + pad), float("nan"), device="cuda") for _ in range(parts)]
    partial_scatter(p, outs, N + pad)
    torch.cuda.synchronize()
    nat.check()
    return p, outs


def _legacy_table(name: str) -> torch.Tensor:
    if name == "fp4":
        from bitsandbytes_b200.functional import get_4bit_type

        return get_4bit_type("fp4", device="cuda")
    g = torch.Generator(device="cpu").manual_seed(30)
    steps = torch.rand(16, generator=g, dtype=torch.float64) + 0.05
    table = torch.cumsum(steps, 0)
    return ((table - table[5]) / table.abs().max()).float().cuda()  # ascending, signed, not a code book


def launch_legacy(table, dtype, K, N, bs, seed):
    """cgemm_4bit_inference_naive_<dtype> on one token with the caller's code table."""
    p = make_problem(1, N, K, "nf4", dtype, bs=bs, seed=seed)
    lut = _legacy_table(table)
    out = torch.full((N,), float("nan"), device="cuda", dtype=nat.DTYPE[dtype])
    fn = getattr(nat.lib, f"cgemm_4bit_inference_naive_{dtype}")
    fn(N, 1, K, p["x"].data_ptr(), p["packed"].data_ptr(), p["absmax"].data_ptr(), lut.data_ptr(), out.data_ptr(), N,
       N, N, bs, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    return p, lut, out


LAUNCHERS = {"routes": launch_routes, "fallback": launch_fallback, "matmul": launch_matmul, "plain": launch_plain,
             "scatter": launch_scatter, "legacy": launch_legacy}


def launch(case):
    kind, kwargs = case
    return LAUNCHERS[kind](**kwargs)


# ----------------------------------------------------------------------- the launch record (a profiled child)
def _arg(a: str) -> str:
    a = re.sub(r"^\((?:bool|int)\)", "", a.strip())
    return {"false": "0", "true": "1"}.get(a, a)


def _instance(name: str):
    """[kernel, template arguments...] of a 4-bit GEMM kernel's demangled name, or None for any other kernel."""
    m = re.search(r"(gemv4_\w+?_kernel)<([^<>]*)>", name)
    if m:
        return [m.group(1)] + [_arg(a) for a in m.group(2).split(",")]
    m = re.search(r"\w*gemm4\w*", name)
    return [m.group(0)] if m else None


def _profiled(fn):
    """The CUDA kernels of one torch.profiler session around fn(), in launch order."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)  # (the first kernels of a session can go unrecorded)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return sorted(kernels, key=lambda e: e.time_range.start)


def record_launches_main():
    """The child: reads a JSON list of cases on stdin, prints one line "LAUNCHES <json>" mapping each case's key to
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
                    got = [i for i in (_instance(e.name) for e in kernels) if i is not None]
                    break
        except Exception as e:  # reported by the test of this case
            got = f"{type(e).__name__}: {e}"
        record[case_key(case)] = got
    print("LAUNCHES " + json.dumps(record), flush=True)


def case_key(case) -> str:
    return json.dumps(case, sort_keys=True)


@pytest.fixture(scope="module")
def launches():
    """{case key: the instances its launches ran}, recorded once for every test of this file by the profiled child."""
    cases = all_cases()
    code = (f"import sys; sys.path.insert(0, {str(ROOT)!r}); "
            "from tests.test_gpu_gemm4_cuda_core import record_launches_main; record_launches_main()")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], input=json.dumps(cases), capture_output=True, text=True,
                       cwd=str(ROOT), timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("LAUNCHES ")]
    if r.returncode != 0 or not lines:
        pytest.fail(f"the profiled child exited with {r.returncode}:\n{r.stderr[-4000:]}")
    return json.loads(lines[-1][len("LAUNCHES "):])


def recorded(launches, case):
    """The instances the case launched, as tuples; skips (only the caller's last assertion) without a record."""
    got = launches[case_key(case)]
    if got is None:
        pytest.skip("torch.profiler recorded no CUDA kernels here: which kernel instance ran is not confirmed")
    assert not isinstance(got, str), f"the profiled replay of this case failed: {got}"
    return [tuple(i) for i in got]


def fast(dtype, qt, mb, part):
    return ("gemv4_fast_kernel", T_NAME[dtype], QT_ARG[qt], str(mb), str(int(part)))


def simt(dtype, part, vec):
    return ("gemv4_simt_kernel", T_NAME[dtype], str(int(part)), str(int(vec)))


def mma(dtype, qt, w, nt, part):
    return ("gemv4_mma_kernel", T_NAME[dtype], QT_ARG[qt], str(w), str(nt), str(int(part)))


# ------------------------------------------------------------------------------ a. gemv4_fast_kernel, every MB
# (M, K, blocksize, nested, bias): K % 32 == 0 but K % 64 != 0, so path 2 at every M; 4192 = 4096 + 32 * 3 leaves a
# tail after the 4 x 1024 step
FAST_ROWS = [
    pytest.param(1, 96, 32, False, True, id="MB1-M1-K96-bs32-bias"),
    pytest.param(2, 160, 64, True, False, id="MB2-M2-K160-bs64-nested"),
    pytest.param(3, 4128, 4096, True, True, id="MB4-M3-K4128-bs4096-nested-bias"),
    pytest.param(4, 4192, 32, False, False, id="MB4-M4-K4192-bs32"),
    pytest.param(5, 4192, 4096, False, True, id="MB8-M5-K4192-bs4096-bias"),
    pytest.param(8, 4128, 32, True, False, id="MB8-M8-K4128-bs32-nested"),
    pytest.param(8, 96, 64, True, True, id="MB8-M8-K96-bs64-nested-bias"),
]


FAST_MB = {1: 1, 2: 2, 3: 4, 4: 4, 5: 8, 8: 8}


def fast_case(M, K, bs, nested, bias, qt, dtype):
    return ["routes", dict(dtype=dtype, M=M, N=203, K=K, bs=bs, qt=qt, nested=nested, bias=bias, seed=21)]


@pytest.mark.parametrize("dtype", DT16)
@pytest.mark.parametrize("qt", QTS)
@pytest.mark.parametrize("M,K,bs,nested,bias", FAST_ROWS)
def test_fast_gemv_every_instance(launches, M, K, bs, nested, bias, qt, dtype):
    """gemv4_fast_kernel<T, QT, MB, PART> for MB in {1, 2, 4, 8}, NF4 and FP4, fp16 and bf16, plain and PART: the
    unforced call takes path 2, equals the call forced to path 0 bit for bit, and meets the oracle bound."""
    case = fast_case(M, K, bs, nested, bias, qt, dtype)
    N = case[1]["N"]  # ragged against the 8 output features of a CTA
    assert nat.lib.cbnb_b200_gemm_4bit_path(M, N, K, bs, nat.DTYPE_ID[dtype]) == 2
    p, out, part = launch(case)
    with forced(0):
        want = run(nat.lib, p)
    nat.check()
    assert torch.equal(run(nat.lib, p).view(torch.int16), want.view(torch.int16))
    check_plain_and_partial(p, out, part)
    mb = FAST_MB[M]
    assert recorded(launches, case) == [fast(dtype, qt, mb, False), fast(dtype, qt, mb, True)]


# ------------------------------------------------------------------------ b. gemv4_simt_kernel, the vector body
# (dtype, M, N, K, blocksize, qt, nested, bias, codes offset in bytes)
VECTOR_ROWS = [
    pytest.param("bf16", 1, 100, 72, 64, "nf4", False, True, 0, id="vector-bf16-M1-K72"),
    pytest.param("fp16", 3, 100, 200, 64, "fp4", True, False, 0, id="vector-fp16-M3-K200-nested"),
    pytest.param("bf16", 9, 100, 4000, 64, "fp4", False, True, 0, id="vector-bf16-M9-K4000"),
    pytest.param("fp16", 37, 72, 4000, 128, "nf4", True, True, 0, id="vector-fp16-M37-K4000-nested"),
    pytest.param("bf16", 300, 40, 4000, 32, "nf4", True, False, 0, id="vector-bf16-M300-K4000-bs32-nested"),
    pytest.param("fp16", 1000, 40, 4000, 64, "fp4", False, True, 0, id="vector-fp16-M1000-K4000"),
    pytest.param("bf16", 2, 100, 96, 48, "nf4", False, True, 0, id="vector-bf16-M2-K96-bs48"),
    pytest.param("fp16", 7, 64, 144, 48, "fp4", True, True, 0, id="vector-fp16-M7-K144-bs48-nested"),
    # codes at a 4-byte, not 16-byte, offset: the fast, mma and wgmma kernels refuse them (paths 2, 3 and 1 unforced)
    pytest.param("bf16", 1, 136, 256, 64, "nf4", False, True, 4, id="vector-bf16-M1-codes+4"),
    pytest.param("fp16", 5, 136, 256, 64, "fp4", True, False, 4, id="vector-fp16-M5-codes+4"),
    pytest.param("bf16", 300, 136, 256, 64, "nf4", True, True, 4, id="vector-bf16-M300-codes+4"),
    # fp32 activations at default precision: the CUDA-core route at every M, K % 64 == 0 included
    pytest.param("fp32", 1, 136, 256, 64, "nf4", False, True, 0, id="vector-fp32-M1"),
    pytest.param("fp32", 4, 136, 512, 64, "fp4", True, False, 0, id="vector-fp32-M4-nested"),
    pytest.param("fp32", 300, 136, 192, 128, "nf4", True, True, 0, id="vector-fp32-M300-nested"),
    pytest.param("fp32", 4096, 72, 256, 64, "fp4", False, True, 0, id="vector-fp32-M4096"),
]




def vector_case(dtype, M, N, K, bs, qt, nested, bias, codes_off):
    return ["routes", dict(dtype=dtype, M=M, N=N, K=K, bs=bs, qt=qt, nested=nested, bias=bias, seed=22,
                           codes_off=codes_off)]


@pytest.mark.parametrize("dtype,M,N,K,bs,qt,nested,bias,codes_off", VECTOR_ROWS)
def test_cuda_core_kernel_vector_body(launches, precision, dtype, M, N, K, bs, qt, nested, bias, codes_off):
    """gemv4_simt_kernel<T, PART, VEC = 1> for fp32, fp16 and bf16, plain and PART: K % 8 == 0 shapes that the fast
    kernel does not take (K % 32 != 0, M > 8, blocksize 48, codes 4-byte aligned only, fp32), partial 4-token groups."""
    precision("ieee")
    case = vector_case(dtype, M, N, K, bs, qt, nested, bias, codes_off)
    check_plain_and_partial(*launch(case))
    assert recorded(launches, case) == [simt(dtype, False, True), simt(dtype, True, True)]


# ------------------------------------------------------------------------ c. gemv4_simt_kernel, the scalar body
# (dtype, M, N, K, blocksize, qt, nested, bias, activation offset in elements, codes offset in bytes).  Odd K with
# N * K a multiple of the blocksize: quantisation blocks span rows, and every other row starts mid-byte.
SCALAR_ROWS = [
    pytest.param("fp32", 3, 64, 1, 64, "nf4", False, True, 0, 0, id="scalar-fp32-M3-K1"),
    pytest.param("bf16", 7, 64, 63, 64, "fp4", True, True, 0, 0, id="scalar-bf16-M7-K63-nested"),
    pytest.param("fp16", 9, 64, 1001, 64, "nf4", False, True, 0, 0, id="scalar-fp16-M9-K1001"),
    pytest.param("fp32", 13, 64, 1001, 64, "fp4", True, False, 0, 0, id="scalar-fp32-M13-K1001-nested"),
    pytest.param("bf16", 37, 64, 63, 64, "fp4", True, True, 0, 0, id="scalar-bf16-M37-K63-nested"),
    pytest.param("bf16", 2, 16, 99, 48, "nf4", False, True, 0, 0, id="scalar-bf16-M2-K99-bs48"),
    pytest.param("fp32", 6, 32, 99, 48, "fp4", True, True, 0, 0, id="scalar-fp32-M6-K99-bs48-nested"),
    pytest.param("fp16", 4, 96, 128, 64, "fp4", True, True, 0, 1, id="scalar-fp16-M4-codes+1"),
    pytest.param("fp32", 5, 96, 128, 32, "nf4", False, True, 0, 1, id="scalar-fp32-M5-codes+1"),
    pytest.param("fp16", 3, 96, 256, 64, "nf4", True, True, 1, 0, id="scalar-fp16-M3-A+1"),
    pytest.param("fp32", 17, 96, 256, 64, "fp4", False, True, 1, 0, id="scalar-fp32-M17-A+1"),
    pytest.param("bf16", 11, 96, 256, 128, "nf4", True, False, 1, 0, id="scalar-bf16-M11-A+1"),
]




def scalar_case(dtype, M, N, K, bs, qt, nested, bias, a_off, codes_off):
    return ["routes", dict(dtype=dtype, M=M, N=N, K=K, bs=bs, qt=qt, nested=nested, bias=bias, seed=23, a_off=a_off,
                           codes_off=codes_off)]


@pytest.mark.parametrize("dtype,M,N,K,bs,qt,nested,bias,a_off,codes_off", SCALAR_ROWS)
def test_cuda_core_kernel_scalar_body(launches, precision, dtype, M, N, K, bs, qt, nested, bias, a_off, codes_off):
    """gemv4_simt_kernel<T, PART, VEC = 0> for fp32, fp16 and bf16, plain and PART: odd K, blocksize 48 (the
    division branch), activations at a 1-element offset, codes at a 1-byte offset."""
    precision("ieee")
    case = scalar_case(dtype, M, N, K, bs, qt, nested, bias, a_off, codes_off)
    check_plain_and_partial(*launch(case))
    assert recorded(launches, case) == [simt(dtype, False, False), simt(dtype, True, False)]


# -------------------------------------------------------------------- d. fallbacks into the CUDA-core kernel
FALLBACK_ROWS = [pytest.param(5, 3, id="M5-mma-refuses"), pytest.param(300, 1, id="M300-wgmma-refuses")]


def fallback_case(M, dtype):
    return ["fallback", dict(dtype=dtype, M=M, N=256, K=512, seed=24)]


@pytest.mark.parametrize("dtype", DT16)
@pytest.mark.parametrize("M,path", FALLBACK_ROWS)
def test_misaligned_activations_fall_back_to_the_scalar_body(launches, M, path, dtype):
    """A contiguous activation view at a 1-element offset: the preferred kernel (mma.sync at 5 tokens, wgmma at 300)
    refuses it and gemv4_simt_kernel's scalar body computes it.  The aligned copy takes the preferred kernel; both
    meet the oracle bound (they are different kernels, so they need not agree bit for bit)."""
    case = fallback_case(M, dtype)
    N, K = case[1]["N"], case[1]["K"]
    assert nat.lib.cbnb_b200_gemm_4bit_path(M, N, K, 64, nat.DTYPE_ID[dtype]) == path
    p, misaligned, aligned = launch(case)
    y64 = exact(p)
    assert_close_to_exact(misaligned, y64, dtype, K)
    assert_close_to_exact(aligned, y64, dtype, K)
    got = recorded(launches, case)
    preferred = "gemv4_mma_kernel" if path == 3 else "gemm4"
    assert got[0] == simt(dtype, False, False), got
    assert len(got) >= 2 and all(preferred in k[0] for k in got[1:]), got


MATMUL_CASE = ["matmul", dict(M=300, N=256, K=512, seed=25)]


def test_matmul_4bit_on_a_misaligned_view_takes_the_cuda_core_kernel(launches):
    """The Python layer keeps a contiguous view as it is, so matmul_4bit reaches the same fallback:
    gemv4_simt_kernel<bf16, PART = 0, VEC = 0>."""
    M, N, K = (MATMUL_CASE[1][k] for k in ("M", "N", "K"))
    x, qW, qs, y = launch(MATMUL_CASE)
    y64 = oracle.gemm_4bit(oracle.widen(nat.to_bits(x).reshape(-1), "bf16"), qW.cpu().numpy(),
                           qs.absmax.cpu().numpy(), M, N, K, 64, "nf4", "bf16")
    assert_close_to_exact(y, y64, "bf16", K)
    assert recorded(launches, MATMUL_CASE) == [simt("bf16", False, False)]


# --------------------------------------------------------------------------- e. gemv4_mma_kernel, every instance
def _mma_n(w: int, n_16: int) -> int:
    """An output width that selects W warps per CTA on this device (launch_gemv4_mma): 4 from 3 row tiles of 16
    per SM on (12 warps per SM at 4 warps per CTA), 16 at K >= 4096 with at most 128 row tiles, 8 in between."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if w == 4:
        return 16 * -(-12 * sms // 4) - 8  # ragged last row tile, still ceil(12 * sms / 4) tiles
    if w == 8:
        return 16 * sms + 8  # sms + 1 row tiles; the rows' K stay below 4096
    return n_16


# (W, M, N for W = 16, K, dtype, qt, blocksize, nested, bias)
MMA_ROWS = [
    pytest.param(16, 1, 1024, 4096, "bf16", "nf4", 64, False, True, id="W16-NT1-M1-N1024-K4096"),
    pytest.param(16, 8, 2048, 4160, "fp16", "fp4", 32, True, False, id="W16-NT1-M8-N2048-K4160"),
    pytest.param(16, 5, 1024, 5120, "bf16", "fp4", 128, True, True, id="W16-NT1-M5-N1024-K5120"),
    pytest.param(16, 9, 2048, 4096, "fp16", "nf4", 64, False, True, id="W16-NT2-M9-N2048-K4096"),
    pytest.param(16, 12, 1024, 4160, "bf16", "nf4", 32, True, True, id="W16-NT2-M12-N1024-K4160"),
    pytest.param(16, 16, 2048, 5120, "bf16", "fp4", 64, False, False, id="W16-NT2-M16-N2048-K5120"),
    pytest.param(8, 2, 0, 1024, "bf16", "nf4", 64, True, True, id="W8-NT1-M2"),
    pytest.param(8, 7, 0, 704, "fp16", "fp4", 32, False, True, id="W8-NT1-M7"),
    pytest.param(8, 12, 0, 1024, "fp16", "nf4", 128, True, False, id="W8-NT2-M12"),
    pytest.param(8, 16, 0, 320, "bf16", "fp4", 64, False, True, id="W8-NT2-M16"),
    pytest.param(4, 1, 0, 512, "fp16", "nf4", 64, False, True, id="W4-NT1-M1"),
    pytest.param(4, 8, 0, 256, "bf16", "fp4", 32, True, True, id="W4-NT1-M8"),
    pytest.param(4, 9, 0, 512, "bf16", "nf4", 64, True, False, id="W4-NT2-M9"),
    pytest.param(4, 16, 0, 192, "fp16", "fp4", 128, False, True, id="W4-NT2-M16"),
]




def mma_case(W, M, N16, K, dtype, qt, bs, nested, bias):
    return ["routes", dict(dtype=dtype, M=M, N=_mma_n(W, N16), K=K, bs=bs, qt=qt, nested=nested, bias=bias, seed=26,
                           path=3)]


@pytest.mark.parametrize("W,M,N16,K,dtype,qt,bs,nested,bias", MMA_ROWS)
def test_mma_decode_kernel_every_instance(launches, W, M, N16, K, dtype, qt, bs, nested, bias):
    """gemv4_mma_kernel<T, QT, W, NT, PART> for W in {4, 8, 16} x NT in {1, 2} x {plain, PART}, forced to path 3:
    the T output against the oracle, the partial against the fp32 bound, and T(partial + bias) == the T output."""
    case = mma_case(W, M, N16, K, dtype, qt, bs, nested, bias)
    check_plain_and_partial(*launch(case))
    nt = 1 if M <= 8 else 2
    assert recorded(launches, case) == [mma(dtype, qt, W, nt, False), mma(dtype, qt, W, nt, True)]


# -------------------------------------------------------------- g. the CUDA-core kernel past 65535 token groups
M_BIG = 4 * SIMT_MAX_TOKEN_GROUPS + 9  # 262 149 tokens, a multiple of 3
BIG_LAUNCHES = 2  # 65 538 groups of 4 tokens: one launch of 65 535 groups and one of 3
BIG_FP32 = ["plain", dict(dtype="fp32", M=M_BIG, N=16, K=64, qt="nf4", nested=True, bias=True, seed=27)]
BIG_SCATTER = ["scatter", dict(dtype="fp32", M=M_BIG, N=16, K=64, qt="fp4", nested=True, seed=28, parts=3, pad=2)]
BIG_BF16 = ["plain", dict(dtype="bf16", M=M_BIG, N=16, K=96, qt="nf4", nested=False, bias=True, seed=29)]


def _assert_tail_written(got: torch.Tensor, y64: np.ndarray, dtype: str, K: int):
    tail = got[-16:]
    assert torch.isfinite(tail.float()).all(), "the last token groups were not written"
    assert_close_to_exact(tail, y64[-16:], dtype, K)


def test_cuda_core_kernel_past_the_grid_limit_fp32(launches, precision):
    """fp32 at 262 149 tokens (more 4-token groups than gridDim.y allows), nested statistics and bias:
    gemv4_simt_kernel<float, PART = 0, VEC = 1>, launched twice."""
    precision("ieee")
    p, got = launch(BIG_FP32)
    y64 = exact(p)
    _assert_tail_written(got, y64, "fp32", 64)
    assert_close_to_exact(got, y64, "fp32", 64)
    assert recorded(launches, BIG_FP32) == [simt("fp32", False, True)] * BIG_LAUNCHES


def test_cuda_core_kernel_past_the_grid_limit_partial_scatter(launches, precision):
    """The fp32 partial at 262 149 tokens scattered over 3 destinations of 87 383 rows each (a sequence-parallel
    row layer's partial): gemv4_simt_kernel<float, PART = 1, VEC = 1>, launched twice."""
    precision("ieee")
    N, K = BIG_SCATTER[1]["N"], BIG_SCATTER[1]["K"]
    p, outs = launch(BIG_SCATTER)
    for o in outs:
        assert torch.isnan(o[:, N:]).all(), "wrote past N"
    got = torch.cat([o[:, :N] for o in outs])
    y64 = exact(p)
    assert torch.isfinite(got[-16:]).all(), "the last token groups were not written"
    assert_partial_close(got, y64, K)
    assert recorded(launches, BIG_SCATTER) == [simt("fp32", True, True)] * BIG_LAUNCHES


def test_cuda_core_kernel_past_the_grid_limit_bf16(launches):
    """bf16 with K = 96 (K % 64 != 0: path 2) at 262 149 tokens: gemv4_simt_kernel<bf16, PART = 0, VEC = 1>,
    launched twice."""
    assert nat.lib.cbnb_b200_gemm_4bit_path(M_BIG, 16, 96, 64, nat.DTYPE_ID["bf16"]) == 2
    p, got = launch(BIG_BF16)
    y64 = exact(p)
    _assert_tail_written(got, y64, "bf16", 96)
    assert_close_to_exact(got, y64, "bf16", 96)
    assert recorded(launches, BIG_BF16) == [simt("bf16", False, True)] * BIG_LAUNCHES


# ------------------------------------------------------------------- h. the legacy GEMV entry, a caller's table
LEGACY_ROWS = [pytest.param(dt, K, id=f"{'vector' if K % 8 == 0 else 'scalar'}-{dt}")
               for dt, K in [("bf16", 512), ("fp16", 77), ("fp32", 320), ("fp32", 77), ("fp16", 256), ("bf16", 77)]]
LEGACY_TABLES = ["fp4", "ascending"]


def legacy_case(table, dtype, K):
    return ["legacy", dict(table=table, dtype=dtype, K=K, N=64, bs=64, seed=31)]  # N * K a multiple of bs at odd K


@pytest.mark.parametrize("table", LEGACY_TABLES)
@pytest.mark.parametrize("dtype,K", LEGACY_ROWS)
def test_legacy_gemv_with_a_callers_table(launches, table, dtype, K):
    """cgemm_4bit_inference_naive_{fp16,bf16,fp32} with the caller's 16 code values: out[n] = sum_k x[k] *
    rn_T(fp32(table[c]) * fp32(absmax)), computed here in float64.  gemv4_simt_kernel<T, PART = 0, VEC> runs it: the
    vector body at K % 8 == 0, the scalar body at odd K."""
    case = legacy_case(table, dtype, K)
    N, bs = case[1]["N"], case[1]["bs"]
    p, lut, out = launch(case)
    packed = p["packed"].cpu().long()
    e = torch.arange(N * K)
    codes = torch.where(e % 2 == 0, packed[e // 2] >> 4, packed[e // 2] & 15)
    w32 = lut.cpu()[codes] * p["absmax"].cpu()[e // bs]  # fp32 products, rounded to nearest
    w = w32.to(nat.DTYPE[dtype]).double().view(N, K)
    y64 = (p["x"].cpu().double() @ w.t()).numpy()
    assert_close_to_exact(out.view(1, N), y64, dtype, K)
    assert recorded(launches, case) == [simt(dtype, False, K % 8 == 0)]


# ------------------------------------------------------------------------------------- every case of the file
def all_cases():
    """The case of every test above, in the order the child replays them."""
    cases = [fast_case(*r.values, qt, dt) for r in FAST_ROWS for qt in QTS for dt in DT16]
    cases += [vector_case(*r.values) for r in VECTOR_ROWS]
    cases += [scalar_case(*r.values) for r in SCALAR_ROWS]
    cases += [fallback_case(r.values[0], dt) for r in FALLBACK_ROWS for dt in DT16]
    cases += [MATMUL_CASE]
    cases += [mma_case(*r.values) for r in MMA_ROWS]
    cases += [BIG_FP32, BIG_SCATTER, BIG_BF16]
    cases += [legacy_case(t, *r.values) for r in LEGACY_ROWS for t in LEGACY_TABLES]
    return cases
