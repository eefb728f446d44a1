"""Loader for the native library (the FFI boundary).

Mirrors the role of the reference's ``bitsandbytes/cextension.py`` (reference
cextension.py:22-80 library selection, :90-115 ``BNBNativeLibrary``, :392-405 deferred
error on load failure) with the multi-backend selection collapsed to the single
sm_90a build: ``libbitsandbytes_b200.so`` next to this file.

There is no CPU fallback and no mock that silently succeeds: if the library is missing
or a symbol cannot be resolved, the first native call raises ``RuntimeError`` naming the
file.  After every native call the host layer polls ``cbnb_b200_last_error`` so that a
failed launch raises instead of the reference's ``exit(1)``.
"""
from __future__ import annotations

import ctypes as ct
import logging
import os
from pathlib import Path

logger = logging.getLogger(__name__)

PACKAGE_DIR = Path(__file__).parent
LIBRARY_NAME = "libbitsandbytes_b200.so"
# names the reference tests / HF integrations probe
HIP_ENVIRONMENT = False
BNB_BACKEND = "CUDA"

_VOIDP = ct.c_void_p
_I32 = ct.c_int32


def _signatures():
    """argtypes/restype per exported symbol -- the Python statement of include/bitsandbytes_b200.h."""
    sig = {}
    dts = ("fp32", "bf16", "fp16")
    for d in dts:
        for q in ("", "_nf4", "_fp4"):
            # (code, A, absmax, out, blocksize, n, stream)
            sig[f"cdequantize_blockwise_{d}{q}"] = ([_VOIDP] * 4 + [_I32, _I32, _VOIDP], None)
            # (code, A, absmax, out, blocksize, n)
            sig[f"cquantize_blockwise_{d}{q}"] = ([_VOIDP] * 4 + [_I32, _I32], None)
        # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, blocksize, quant_type, stream)
        sig[f"cgemm_4bit_{d}"] = ([_VOIDP] * 8 + [_I32] * 5 + [_VOIDP], None)
        # (m, n, k, A, B, absmax, code, out, lda, ldb, ldc, blocksize, stream)
        sig[f"cgemm_4bit_inference_naive_{d}"] = ([_I32] * 3 + [_VOIDP] * 5 + [_I32] * 4 + [_VOIDP], None)
    sig["get_context"] = ([], _VOIDP)
    # (ctx, m, n, k, A, B, C, row_scale, lda, ldb, ldc, stream) -> int
    sig["cigemmlt_32"] = ([_VOIDP] + [_I32] * 3 + [_VOIDP] * 4 + [_I32] * 3 + [_VOIDP], _I32)
    # (A, rowStats, colStats, out, bias, numRows, numCols, stream)
    sig["cdequant_mm_int32_fp16"] = ([_VOIDP] * 5 + [_I32, _I32, _VOIDP], None)
    # (A, out, rowStats, threshold, rows, cols, stream)
    sig["cint8_vector_quant"] = ([_VOIDP] * 3 + [ct.c_float, _I32, _I32, _VOIDP], None)
    # ---- native additions
    sig["cbnb_b200_last_error"] = ([], _I32)
    sig["cbnb_b200_last_error_message"] = ([], ct.c_char_p)
    sig["cbnb_b200_build_info"] = ([], ct.c_char_p)
    # (code, A, absmax, out, blocksize, n, quant_type, dtype, stream)
    sig["cbnb_b200_quantize_blockwise"] = ([_VOIDP] * 4 + [_I32] * 4 + [_VOIDP], None)
    sig["cbnb_b200_gemm_4bit_path"] = ([_I32] * 5, _I32)
    sig["cbnb_b200_gemm_4bit_force_path"] = ([_I32], None)
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, ldc, blocksize, quant_type, dtype, stream)
    sig["cbnb_b200_gemm_4bit_strided"] = ([_VOIDP] * 8 + [_I32] * 7 + [_VOIDP], None)
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, ldc, blocksize, quant_type, dtype,
    #  mt, force_splits, trace, stream) -> int
    sig["cbnb_b200_gemm_4bit_pair"] = ([_VOIDP] * 8 + [_I32] * 9 + [_VOIDP, _VOIDP], _I32)
    sig["cbnb_b200_gemm_4bit_multi_out"] = ([_VOIDP] * 7 + [_I32] + [_VOIDP] + [_I32] * 7 + [_VOIDP], _I32)
    # (CA, CB, SCA, SCB, bias, out, M, N, K, dtype, stream) -> int
    sig["cbnb_b200_int8_scaled_mm"] = ([_VOIDP] * 6 + [_I32] * 4 + [_VOIDP], _I32)
    # (CA, CB, SCA, SCB, bias, subA, subBT, jpad, out, M, N, K, dtype, stream) -> int
    sig["cbnb_b200_int8_mixed_mm"] = ([_VOIDP] * 7 + [_I32] + [_VOIDP] + [_I32] * 4 + [_VOIDP], _I32)
    # (A, CB, SCB, cols, J, jpad, M, N, K, dtype, subA, subBT, stream)
    sig["cbnb_b200_int8_outlier_prep"] = ([_VOIDP] * 4 + [_I32] * 6 + [_VOIDP] * 3, None)
    # (A, out, col_stats, threshold, rows, cols, dtype, stream) -> int
    sig["cbnb_b200_int8_col_quant"] = ([_VOIDP] * 3 + [ct.c_float] + [_I32] * 3 + [_VOIDP], _I32)
    # (CA, cols, J, rows, K, stream)
    sig["cbnb_b200_int8_zero_columns"] = ([_VOIDP] * 2 + [_I32] * 3 + [_VOIDP], None)
    # (A, out, rowStats, col_flags, threshold, rows, cols, dtype, stream)
    sig["cbnb_b200_int8_vector_quant_flags"] = ([_VOIDP] * 4 + [ct.c_float] + [_I32] * 3 + [_VOIDP], None)
    # (A, B, value, n)
    sig["cfill_fp32"] = ([_VOIDP, _VOIDP, ct.c_float, ct.c_long], None)
    sig["cfill_uint8"] = ([_VOIDP, _VOIDP, ct.c_ubyte, ct.c_long], None)
    sig["carange_fp32"] = ([_VOIDP, _VOIDP, ct.c_float, ct.c_long], None)
    sig["c_mul_fp32"] = ([_VOIDP, _VOIDP, ct.c_float, ct.c_long], None)
    sig["cget_managed_ptr"] = ([ct.c_size_t], _VOIDP)
    sig["cprefetch"] = ([_VOIDP, ct.c_size_t, _I32], None)
    # ---- optimizers (SURVEY.md section 8 row f-4)
    _F = ct.c_float
    # (g, p, state1, state2, unorm, max_unorm, param_norm, beta1, beta2, beta3, alpha, eps, weight_decay, step, lr,
    #  gnorm_scale, skip_zeros, n)
    sig32 = ([_VOIDP] * 5 + [_F] * 8 + [_I32, _F, _F, ct.c_bool, _I32], None)
    for name, sufs in (("adam", ("fp32", "fp16", "bf16")), ("lion", ("fp32", "fp16", "bf16")),
                       ("ademamix", ("fp32", "fp16", "bf16")), ("momentum", ("32", "16")), ("rmsprop", ("32", "16")),
                       ("adagrad", ("32", "16"))):
        for suf in sufs:
            sig[f"c{name}32bit_grad_{suf}"] = sig32
    # (p, g, state1, state2, beta1, beta2, beta3, alpha, eps, step, lr, quantiles1, quantiles2, absmax1, absmax2,
    #  weight_decay, gnorm_scale, skip_zeros, n)
    sig8 = ([_VOIDP] * 4 + [_F] * 5 + [_I32, _F] + [_VOIDP] * 4 + [_F, _F, ct.c_bool, _I32], None)
    for name in ("adam", "momentum", "rmsprop", "adagrad", "lion", "ademamix"):
        for suf in ("fp32", "fp16", "bf16"):
            sig[f"c{name}_8bit_blockwise_grad_{suf}"] = sig8
    # (optimizer, dtype, g, p, state1, state2, unorm, max_unorm .. gnorm_scale, skip_zeros, n, stream) -> int
    sig["cbnb_b200_optimizer_update_32bit"] = ([_I32, _I32] + [_VOIDP] * 5 + [_F] * 8 + [_I32, _F, _F, ct.c_bool,
                                                ct.c_longlong, _VOIDP], _I32)
    # (optimizer, dtype, p, g, state1, state2, beta1 .. eps, step, lr, q1, q2, absmax1, absmax2, weight_decay,
    #  gnorm_scale, skip_zeros, n, stream) -> int
    sig["cbnb_b200_optimizer_update_8bit_blockwise"] = ([_I32, _I32] + [_VOIDP] * 4 + [_F] * 5 + [_I32, _F] + [_VOIDP] * 4
                                                        + [_F, _F, ct.c_bool, ct.c_longlong, _VOIDP], _I32)
    return sig


EXPORTED_SYMBOLS = tuple(sorted(_signatures()))


class NativeLibraryError(RuntimeError):
    pass


class _Missing:
    """Stands in for the library when it cannot be loaded: every use raises, loudly."""

    def __init__(self, reason: str):
        self._reason = reason

    def __getattr__(self, name):
        raise NativeLibraryError(
            f"bitsandbytes_b200 native library unavailable ({self._reason}); "
            f"build it with `python -c 'import __graft_entry__ as g; g.build()'` or "
            f"`make -C bitsandbytes_b200/csrc`. There is no CPU or PyTorch fallback."
        )


class NativeLibrary:
    compiled_with_cuda = True

    def __init__(self, dll: ct.CDLL, path: Path):
        self._dll = dll
        self.path = path
        for name, (argtypes, restype) in _signatures().items():
            try:
                fn = getattr(dll, name)
            except AttributeError as e:  # a symbol the header declares is absent: the build is broken
                raise NativeLibraryError(f"{path} does not export {name}") from e
            fn.argtypes = argtypes
            fn.restype = restype
            setattr(self, name, fn)

    def check(self, what: str = "native call") -> None:
        code = self.cbnb_b200_last_error()
        if code != 0:
            msg = self.cbnb_b200_last_error_message()
            raise RuntimeError(f"{what}: {msg.decode() if msg else 'unknown error'} (code {code})")

    def build_info(self) -> str:
        return self.cbnb_b200_build_info().decode()


def library_path() -> Path:
    override = os.environ.get("BNB_B200_LIBRARY")
    return Path(override) if override else PACKAGE_DIR / LIBRARY_NAME


def get_native_library():
    path = library_path()
    if not path.exists():
        logger.warning("bitsandbytes_b200: %s not found", path)
        return _Missing(f"{path} not found")
    try:
        dll = ct.cdll.LoadLibrary(str(path))
    except OSError as e:
        logger.warning("bitsandbytes_b200: failed to load %s: %s", path, e)
        return _Missing(f"dlopen({path}) failed: {e}")
    return NativeLibrary(dll, path)


lib = get_native_library()
