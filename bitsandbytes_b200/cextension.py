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
    sig["cbnb_b200_gemm_4bit_staged_route"] = ([_I32] * 5, _I32)
    sig["cbnb_b200_gemm_4bit_force_path"] = ([_I32], None)
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, ldc, blocksize, quant_type, dtype, stream)
    # dtype for the 4-bit GEMM entries: 0 fp32, 1 fp16, 2 bf16, 3 fp32 with TF32 allowed
    sig["cbnb_b200_gemm_4bit_strided"] = ([_VOIDP] * 8 + [_I32] * 7 + [_VOIDP], None)
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, ldc, blocksize, quant_type, dtype,
    #  mt, force_splits, trace, stream) -> int
    sig["cbnb_b200_gemm_4bit_pair"] = ([_VOIDP] * 8 + [_I32] * 9 + [_VOIDP, _VOIDP], _I32)
    sig["cbnb_b200_gemm_4bit_multi_out"] = ([_VOIDP] * 7 + [_I32] + [_VOIDP] + [_I32] * 7 + [_VOIDP], _I32)
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, outs, n_outs, M, N, K, ldc, blocksize, quant_type, dtype,
    #  stream) -> int
    sig["cbnb_b200_gemm_4bit_partial"] = ([_VOIDP] * 7 + [_I32] * 8 + [_VOIDP], _I32)
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, outs, n_outs, rows_per_out, M, N, K, ldc, blocksize,
    #  quant_type, dtype, stream) -> int
    sig["cbnb_b200_gemm_4bit_partial_scatter"] = ([_VOIDP] * 7 + [_I32] * 9 + [_VOIDP], _I32)
    # (parts, world, part_stride, out, bias, M, N, ldc, dtype, stream) -> int
    sig["cbnb_b200_reduce_partials"] = ([_VOIDP, _I32, ct.c_longlong, _VOIDP, _VOIDP] + [_I32] * 4 + [_VOIDP], _I32)
    # (parts, n_parts, row0, rows, out, bias, M, N, ldc, dtype, stream) -> int
    sig["cbnb_b200_reduce_partials_ptrs"] = ([_VOIDP] + [_I32] * 3 + [_VOIDP] * 2 + [_I32] * 4 + [_VOIDP], _I32)
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, outs, n_outs, bias, M, N, K, ldc, blocksize, quant_type,
    #  dtype, mt, panel_rows, stream) -> int
    sig["cbnb_b200_gemm_4bit_staged"] = ([_VOIDP] * 7 + [_I32] + [_VOIDP] + [_I32] * 9 + [_VOIDP], _I32)
    # (A, B, absmax, absmax_8bit, absmax_code, absmax_offset, offs, E, out, bias, M, N, K, ldc, blocksize, quant_type,
    #  dtype, stream) -> int; the _mt form takes mt before the stream
    sig["cbnb_b200_gemm_4bit_grouped"] = ([_VOIDP] * 7 + [_I32] + [_VOIDP] * 2 + [_I32] * 7 + [_VOIDP], _I32)
    sig["cbnb_b200_gemm_4bit_grouped_mt"] = ([_VOIDP] * 7 + [_I32] + [_VOIDP] * 2 + [_I32] * 8 + [_VOIDP], _I32)
    # (A, B, absmax, offs, E, out, M, N, K, ldc, blocksize, quant_type, dtype, mt, stream) -> int
    sig["cbnb_b200_gemm_4bit_grouped_partial"] = ([_VOIDP] * 4 + [_I32] + [_VOIDP] + [_I32] * 8 + [_VOIDP], _I32)
    # (parts, world, part_stride, offs, E, out, bias, M, N, ldc, dtype, stream) -> int
    sig["cbnb_b200_reduce_partials_grouped"] = ([_VOIDP, _I32, ct.c_longlong, _VOIDP, _I32, _VOIDP, _VOIDP] + [_I32] * 4
                                                + [_VOIDP], _I32)
    # (B, absmax, absmax_8bit, absmax_code, absmax_offset, out, blocksize, quant_type, dtype, n0, rows, K, stream) -> int
    sig["cbnb_b200_dequantize_4bit_panel"] = ([_VOIDP] * 6 + [_I32] * 6 + [_VOIDP], _I32)
    # (A, W, out, bias, M, N, K, ldc, dtype, mt, stream) -> int
    sig["cbnb_b200_gemm_decoded"] = ([_VOIDP] * 4 + [_I32] * 6 + [_VOIDP], _I32)
    # (CA, CB, SCA, SCB, bias, out, M, N, K, dtype, stream) -> int
    sig["cbnb_b200_int8_scaled_mm"] = ([_VOIDP] * 6 + [_I32] * 4 + [_VOIDP], _I32)
    # (CA, CB, SCA, SCB, bias, subA, subBT, jpad, out, M, N, K, dtype, stream) -> int
    sig["cbnb_b200_int8_mixed_mm"] = ([_VOIDP] * 7 + [_I32] + [_VOIDP] + [_I32] * 4 + [_VOIDP], _I32)
    # (A, CB, SCB, cols, J, jpad, M, N, K, dtype, subA, subBT, stream)
    sig["cbnb_b200_int8_outlier_prep"] = ([_VOIDP] * 4 + [_I32] * 6 + [_VOIDP] * 3, None)
    # (A, out, col_stats, threshold, rows, cols, dtype, stream) -> int
    sig["cbnb_b200_int8_col_quant"] = ([_VOIDP] * 3 + [ct.c_float] + [_I32] * 3 + [_VOIDP], _I32)
    # (CB, SCB, out, ldo, rows, cols, dtype, stream) -> int
    sig["cbnb_b200_int8_dequant_rows"] = ([_VOIDP] * 3 + [_I32] * 4 + [_VOIDP], _I32)
    # (CA, cols, J, rows, K, stream)
    sig["cbnb_b200_int8_zero_columns"] = ([_VOIDP] * 2 + [_I32] * 3 + [_VOIDP], None)
    # (col_flags, K, cols, count, stream)
    sig["cbnb_b200_int8_outlier_compact"] = ([_VOIDP, _I32, _VOIDP, _VOIDP, _VOIDP], None)
    # (A, CA, CB, SCB, cols, count, M, N, K, dtype, subA, subBT, stream)
    sig["cbnb_b200_int8_outlier_prep_dev"] = ([_VOIDP] * 6 + [_I32] * 4 + [_VOIDP] * 3, None)
    # (CA, CB, SCA, SCB, bias, A, subA, subBT, cols, count, out, M, N, K, dtype, stream) -> int
    sig["cbnb_b200_int8_mixed_mm_dev"] = ([_VOIDP] * 11 + [_I32] * 4 + [_VOIDP], _I32)
    # (A, A16, CA, CB, SCB, offs, E, threshold, ends, flags, cols, count, subA, subBT, M, N, K, dtype, stream) -> int
    sig["cbnb_b200_int8_grouped_outliers"] = ([_VOIDP] * 6 + [_I32, ct.c_float] + [_VOIDP] * 6 + [_I32] * 4 + [_VOIDP],
                                              _I32)
    # (CA, CB, SCA, SCB, bias, offs, E, A, subA, subBT, cols, count, out, M, N, K, dtype, stream) -> int
    sig["cbnb_b200_int8_grouped_mm"] = ([_VOIDP] * 6 + [_I32] + [_VOIDP] * 6 + [_I32] * 4 + [_VOIDP], _I32)
    # (A, out, rowStats, col_flags, threshold, rows, cols, dtype, stream)
    sig["cbnb_b200_int8_vector_quant_flags"] = ([_VOIDP] * 4 + [ct.c_float] + [_I32] * 3 + [_VOIDP], None)
    # (A, rowStats, col_flags, threshold, rows, cols, dtype, stream) -> int
    sig["cbnb_b200_int8_row_stats"] = ([_VOIDP] * 3 + [ct.c_float] + [_I32] * 3 + [_VOIDP], _I32)
    # (A, out, rowStats, threshold, rows, cols, dtype, stream) -> int
    sig["cbnb_b200_int8_quant_with_stats"] = ([_VOIDP] * 3 + [ct.c_float] + [_I32] * 3 + [_VOIDP], _I32)
    # (CA, CB, SCA, SCB, bias, subA, subBT, jpad, outs, n_outs, M, N, K, ldc, epi, stream) -> int
    sig["cbnb_b200_int8_gemm_multi_out"] = ([_VOIDP] * 7 + [_I32, _VOIDP] + [_I32] * 6 + [_VOIDP], _I32)
    # (CA, CB, outs, n_outs, rows_per_out, M, N, K, ldc, stream) -> int
    sig["cbnb_b200_int8_gemm_partial_scatter"] = ([_VOIDP] * 3 + [_I32] * 6 + [_VOIDP], _I32)
    # (parts, world, part_stride, SCA, SCB, bias, subA, subBT, jpad, out, M, N, ldc, dtype, stream) -> int
    sig["cbnb_b200_int8_reduce_partials"] = ([_VOIDP, _I32, ct.c_longlong] + [_VOIDP] * 5 + [_I32, _VOIDP] + [_I32] * 4
                                             + [_VOIDP], _I32)
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
    sig["cbnb_b200_optimizer_multi_capacity"] = ([], _I32)
    # (optimizer, dtype, tensors (bnb_b200_optim_tensor_t[count]), count, beta1, beta2, beta3, alpha, eps, weight_decay,
    #  lr, gnorm_scale, skip_zeros, stream) -> int
    sig["cbnb_b200_optimizer_update_32bit_multi"] = ([_I32, _I32, _VOIDP, _I32] + [_F] * 8 + [ct.c_bool, _VOIDP], _I32)
    # (optimizer, dtype, tensors, count, beta1, beta2, beta3, alpha, eps, weight_decay, lr, q1, q2, gnorm_scale,
    #  skip_zeros, stream) -> int
    sig["cbnb_b200_optimizer_update_8bit_blockwise_multi"] = ([_I32, _I32, _VOIDP, _I32] + [_F] * 7 + [_VOIDP, _VOIDP, _F,
                                                               ct.c_bool, _VOIDP], _I32)
    # the capturable forms: (optimizer, dtype, tensors (with step_ptr), count, beta1 .. lr, lr_dev, ...) -> int
    sig["cbnb_b200_optimizer_update_32bit_multi_dev"] = ([_I32, _I32, _VOIDP, _I32] + [_F] * 7 + [_VOIDP, _F, ct.c_bool,
                                                          _VOIDP], _I32)
    sig["cbnb_b200_optimizer_update_8bit_blockwise_multi_dev"] = ([_I32, _I32, _VOIDP, _I32] + [_F] * 7 + [_VOIDP] * 3
                                                                   + [_F, ct.c_bool, _VOIDP], _I32)
    # the data-parallel forms: (optimizer, dtype, tensors, count, grad_srcs, world, param_dsts, ndst, grad_local,
    #  param_local, numel, grad_scale, beta1 .. lr, [q1, q2,] skip_zeros, stream) -> int
    sig["cbnb_b200_optimizer_peers_capacity"] = ([], _I32)
    peers = [_I32, _I32, _VOIDP, _I32, _VOIDP, _I32, _VOIDP, _I32, _VOIDP, _VOIDP, ct.c_longlong] + [_F] * 8
    sig["cbnb_b200_optimizer_update_32bit_multi_peers"] = (peers + [ct.c_bool, _VOIDP], _I32)
    sig["cbnb_b200_optimizer_update_8bit_blockwise_multi_peers"] = (peers + [_VOIDP, _VOIDP, ct.c_bool, _VOIDP], _I32)
    # the clipped forms: (... skip_zeros, gnorm_scale_dev, stream) -> int
    sig["cbnb_b200_optimizer_update_32bit_multi_peers_scaled"] = (peers + [ct.c_bool, _VOIDP, _VOIDP], _I32)
    sig["cbnb_b200_optimizer_update_8bit_blockwise_multi_peers_scaled"] = (peers + [_VOIDP, _VOIDP, ct.c_bool, _VOIDP,
                                                                                    _VOIDP], _I32)
    # the capturable forms (descriptors with step_ptr): (... skip_zeros, gnorm_scale_dev, lr_dev, stream) -> int
    sig["cbnb_b200_optimizer_update_32bit_multi_peers_dev"] = (peers + [ct.c_bool] + [_VOIDP] * 3, _I32)
    sig["cbnb_b200_optimizer_update_8bit_blockwise_multi_peers_dev"] = (peers + [_VOIDP, _VOIDP, ct.c_bool]
                                                                        + [_VOIDP] * 3, _I32)
    # (dtype, tensors, count, grad_srcs, world, grad_local, numel, grad_scale, inf_norm, acc, stream) -> int
    sig["cbnb_b200_optimizer_grad_norm_peers"] = ([_I32, _VOIDP, _I32, _VOIDP, _I32, _VOIDP, ct.c_longlong, _F,
                                                   ct.c_bool, _VOIDP, _VOIDP], _I32)
    # (rank_values, world, inf_norm, max_norm, out, stream) -> int
    sig["cbnb_b200_optimizer_clip_coef"] = ([_VOIDP, _I32, ct.c_bool, _F, _VOIDP, _VOIDP], _I32)
    return sig


class OptimTensor(ct.Structure):
    """One entry of a multi-tensor optimizer call: bnb_b200_optim_tensor_t of include/bitsandbytes_b200.h.

    ``step`` and ``reserved`` share their 8 bytes with ``step_ptr``, the device step counter of the capturable (_dev)
    entries: the C union, which ctypes fields cannot overlap, is the ``step_ptr`` property."""

    _fields_ = [("p", _VOIDP), ("g", _VOIDP), ("state1", _VOIDP), ("state2", _VOIDP), ("absmax1", _VOIDP),
                ("absmax2", _VOIDP), ("n", ct.c_longlong), ("step", ct.c_int32), ("reserved", ct.c_int32)]

    @property
    def step_ptr(self):
        return _VOIDP.from_buffer(self, OptimTensor.step.offset).value

    @step_ptr.setter
    def step_ptr(self, ptr):
        _VOIDP.from_buffer(self, OptimTensor.step.offset).value = ptr


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
