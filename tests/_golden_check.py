"""Shared checker: run a quantize / dequantize implementation over the reference-generated golden
vectors (tests/golden/reference_vectors_*.npz).  The GPU suite passes the C-ABI calls of the product
library; the CPU suite passes the oracle, which validates this checker itself.

quantize_fn(A_bits_or_f32: np.ndarray, dtype: str, blocksize, qt, code) -> (codes u8, absmax f32)
dequantize_fn(codes u8, absmax f32, blocksize, n, qt, code, out_dtype: str) -> np.ndarray of bit patterns
(uint16 for bf16/fp16, float32 viewed as uint32 for fp32)."""
from pathlib import Path

import numpy as np

GOLDEN_DIR = Path(__file__).resolve().parent / "golden"
Q8_NAMES = ["a", "b", "c", "d", "e", "f", "g", "h"]
Q4_NAMES = ["a", "b", "c", "d", "e", "f", "g", "h", "i"]
OUT_DTYPES = ["fp32", "bf16", "fp16"]


def load():
    """All arrays of the golden set (stored in parts of under 1 MB each) as one dict."""
    out = {}
    for part in sorted(GOLDEN_DIR.glob("reference_vectors_*.npz")):
        with np.load(part) as z:
            out.update({k: z[k] for k in z.files})
    return out


def _canon_zero(bits: np.ndarray) -> np.ndarray:
    """+0 and -0 compare equal (FP4 has two zeros: the CUDA kernels keep the sign, the CPU ones do not)."""
    b = bits.copy()
    if b.dtype == np.uint16:
        b[b == 0x8000] = 0
    else:
        b[b == 0x80000000] = 0
    return b


def _as_bits(x: np.ndarray) -> np.ndarray:
    return x.view(np.uint32) if x.dtype == np.float32 else x.view(np.uint16)


def check_8bit(z, name, quantize_fn, dequantize_fn):
    A = z[f"q8_{name}_A"]
    bs = int(z[f"q8_{name}_bs"])
    code = z["dynamic_map"]
    n = A.size
    codes, absmax = quantize_fn(A, "fp32", bs, None, code)
    np.testing.assert_array_equal(absmax, z[f"q8_{name}_absmax"], err_msg="absmax must be bit-exact")
    ref_codes = z[f"q8_{name}_codes"].reshape(-1)
    # codes: only inputs within a few ulp of a decision threshold may differ (GPU: MUFU.RCP normalisation)
    differing = int((codes.reshape(-1) != ref_codes).sum())
    assert differing <= max(2, n // 500), f"{differing} of {n} codes differ from the reference"
    for dt in OUT_DTYPES:
        got = dequantize_fn(ref_codes, z[f"q8_{name}_absmax"], bs, n, None, code, dt)
        np.testing.assert_array_equal(_as_bits(got).reshape(-1), _as_bits(z[f"q8_{name}_deq_{dt}_default"]).reshape(-1),
                                      err_msg=f"dequantize -> {dt} must be bit-exact")


def check_4bit(z, qt, name, quantize_fn, dequantize_fn):
    key = f"q4_{qt}_{name}"
    dt_in = str(z[f"{key}_dtype"])
    A = z[f"{key}_A"]
    bs = int(z[f"{key}_bs"])
    n = A.size
    packed, absmax = quantize_fn(A.reshape(-1), dt_in, bs, qt, None)
    np.testing.assert_array_equal(absmax, z[f"{key}_absmax"], err_msg="absmax must be bit-exact")
    ref = z[f"{key}_packed"].reshape(-1)
    assert packed.reshape(-1).shape == ref.shape

    def nibbles(p):
        hi, lo = p >> 4, p & 15
        if qt == "fp4":  # the two zeros are the same value
            hi = np.where(hi == 8, 0, hi)
            lo = np.where(lo == 8, 0, lo)
        return np.stack([hi, lo], axis=1).reshape(-1)[:n]

    differing = int((nibbles(packed.reshape(-1)) != nibbles(ref)).sum())
    assert differing <= max(1, n // 200), f"{differing} of {n} 4-bit codes differ from the reference"
    for dt in OUT_DTYPES:
        got = dequantize_fn(ref, z[f"{key}_absmax"], bs, n, qt, None, dt)
        want = z[f"{key}_deq_{dt}_default"].reshape(-1)
        np.testing.assert_array_equal(_canon_zero(_as_bits(got).reshape(-1)), _canon_zero(_as_bits(want)),
                                      err_msg=f"dequantize_4bit -> {dt} must be bit-exact")


GEMM4_NAMES = ["plain", "nested", "fp16"]


def check_gemm4(z, name, gemm_fn):
    """gemm_fn(x_bits u16, dtype, packed u8, absmax f32, absmax_8bit u8|None, absmax_code f32|None,
    absmax_offset float|None, bias_bits u16|None, M, N, K, blocksize, qt) -> [M, N] float64 values of T.
    The golden output is the reference's public API on its CPU backend (dequantize + F.linear in T):
    two roundings of the same exact sums, so within two T-ulps of each other."""
    key = f"gemm4_{name}"
    M, N, K = (int(v) for v in z[f"{key}_shape"])
    qt = str(z[f"{key}_qt"])
    dt = str(z[f"{key}_dtype"])
    nested = f"{key}_absmax8" in z
    absmax = z[f"{key}_absmax2"] if nested else z[f"{key}_absmax"]
    a8 = z[f"{key}_absmax8"] if nested else None
    code2 = z[f"{key}_code2"] if nested else None
    offset = float(z[f"{key}_offset"][0]) if nested else None
    bias = z[f"{key}_bias"] if f"{key}_bias" in z else None
    got = gemm_fn(z[f"{key}_x"].reshape(-1), dt, z[f"{key}_packed"], absmax, a8, code2, offset, bias, M, N, K, 64, qt)
    got = np.asarray(got, dtype=np.float64).reshape(M, N)
    y_bits = z[f"{key}_y"].reshape(-1)
    if dt == "bf16":
        y_ref = (y_bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64).reshape(M, N)
        eps = 2.0**-8
    else:
        y_ref = y_bits.view(np.float16).astype(np.float64).reshape(M, N)
        eps = 2.0**-11
    assert np.all(np.isfinite(got))
    err = np.abs(got - y_ref)
    assert np.all(err <= 2 * eps * np.abs(y_ref) + 4e-3), float(err.max())


def check_int8_gemm(z, gemm_fn, dequant_fn):
    """gemm_fn(A i8 [M,K], B i8 [N,K]) -> int32 [M,N] (exact); dequant_fn(C i32, row_stats, col_stats, bias_bits|None)
    -> fp16 bit patterns [M,N], within one fp16 ulp of the reference's pure-torch kernel (which multiplies by
    1/127^2 in a different order)."""
    C = gemm_fn(z["i8mm_A"], z["i8mm_B"])
    np.testing.assert_array_equal(C, z["i8mm_C"])
    for tag, bias in (("nobias", None), ("bias", z["i8mm_bias"])):
        got = np.asarray(dequant_fn(z["i8mm_C"], z["i8mm_rs"], z["i8mm_cs"], bias)).reshape(-1).view(np.float16)
        want = z[f"i8mm_deq_{tag}"].reshape(-1).view(np.float16)
        ulp = np.spacing(np.abs(want)).astype(np.float32)
        assert np.all(np.abs(got.astype(np.float32) - want.astype(np.float32)) <= ulp + 1e-7)
