"""Host side of the sm_90a kernels: argument checking, output allocation, the ctypes call.

Plays the role of the reference's ``bitsandbytes/backends/cuda/ops.py`` (:78-982) for the
hot path, with three structural differences:

* no per-architecture heuristic (reference :583-811) and no dequantize + cuBLAS fallback
  (:904-916): ``gemm_4bit`` always runs a fused kernel -- wgmma for 16-bit activations,
  CUDA cores for fp32 / odd shapes; the choice is made inside the library;
* ``int8_vectorwise_quant`` finds outlier columns inside the quantisation kernel instead
  of three torch kernels and a host sync (reference :230-236); the data-dependent
  ``outlier_cols`` tensor still has to be materialised (``nonzero``), once;
* ``int8_scaled_mm`` / ``int8_mixed_scaled_mm`` use the int8 wgmma GEMM with the
  dequantisation fused into its epilogue (the reference chains cuBLASLt -> int32 in HBM ->
  an elementwise kernel, backends/default/ops.py:64-119).

Every call polls the library's error flag: a failed launch raises instead of killing the
process.
"""
from __future__ import annotations

import ctypes as ct
from math import prod
from typing import Optional, Sequence
from warnings import warn

import torch

from .._ops import kernel
from ..cextension import lib

_DTYPE_SUFFIX = {torch.float32: "fp32", torch.float16: "fp16", torch.bfloat16: "bf16"}
_DTYPE_ID = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
_QT_ID = {"fp4": 1, "nf4": 2}
_4BIT_BLOCKSIZES = (32, 64, 128, 256, 512, 1024, 2048, 4096)
_8BIT_BLOCKSIZES = (64, 128, 256, 512, 1024, 2048, 4096)

_raw_stream = torch._C._cuda_getCurrentRawStream


_INT32_MAX = 2**31 - 1


def _check_sizes(what: str, *sizes: int) -> None:
    """The C ABI carries element counts and dimensions as 32-bit ints (as the reference's does, reference
    csrc/pythonInterface.cpp:343-616): refuse anything that would wrap instead of processing a prefix silently."""
    for v in sizes:
        if v > _INT32_MAX:
            raise ValueError(f"{what}: size {v} exceeds the 32-bit range of the native interface")


def _stream(t: torch.Tensor) -> int:
    return _raw_stream(t.device.index)


class _on_device:
    """Make the tensor's device current for the call (no-op on single-GPU processes)."""

    __slots__ = ("idx", "prev")

    def __init__(self, t: torch.Tensor):
        self.idx = t.device.index
        self.prev = None

    def __enter__(self):
        if torch.cuda.device_count() > 1:
            cur = torch.cuda.current_device()
            if cur != self.idx:
                self.prev = cur
                torch.cuda.set_device(self.idx)

    def __exit__(self, *exc):
        if self.prev is not None:
            torch.cuda.set_device(self.prev)
        return False


def _suffix(dtype: torch.dtype, what: str) -> str:
    try:
        return _DTYPE_SUFFIX[dtype]
    except KeyError:
        raise ValueError(f"{what} only supports 16/32-bit floats, but got {dtype}") from None


# ====================================================================================== blockwise
@kernel("quantize_blockwise")
def _quantize_blockwise(A: torch.Tensor, code: torch.Tensor, blocksize: int):
    if code.dtype != torch.float32:
        raise ValueError(f"code must be float32, got {code.dtype}")
    if blocksize not in _8BIT_BLOCKSIZES:
        raise ValueError(f"invalid blocksize {blocksize}")
    sfx = _suffix(A.dtype, "Blockwise quantization")
    A = A.contiguous()
    n = A.numel()
    _check_sizes("quantize_blockwise", n)
    absmax = torch.empty((-(n // -blocksize),), device=A.device, dtype=torch.float32)
    out = torch.empty_like(A, dtype=torch.uint8)
    with _on_device(A):
        lib.cbnb_b200_quantize_blockwise(code.data_ptr(), A.data_ptr(), absmax.data_ptr(), out.data_ptr(), blocksize,
                                         n, 0, _DTYPE_ID[A.dtype], _stream(A))
    lib.check(f"quantize_blockwise[{sfx}]")
    return out, absmax


def _dequantize_blockwise_into(A, absmax, code, blocksize, dtype, out) -> None:
    sfx = _suffix(dtype, "Blockwise dequantization")
    A = A.contiguous()
    _check_sizes("dequantize_blockwise", A.numel())
    with _on_device(A):
        getattr(lib, f"cdequantize_blockwise_{sfx}")(code.data_ptr(), A.data_ptr(), absmax.data_ptr(), out.data_ptr(),
                                                     blocksize, A.numel(), _stream(A))
    lib.check(f"dequantize_blockwise[{sfx}]")


@kernel("dequantize_blockwise")
def _dequantize_blockwise(A, absmax, code, blocksize: int, dtype: torch.dtype):
    out = torch.empty_like(A, dtype=dtype)
    _dequantize_blockwise_into(A, absmax, code, blocksize, dtype, out)
    return out


@kernel("dequantize_blockwise.out")
def _dequantize_blockwise_out(A, absmax, code, blocksize: int, dtype: torch.dtype, out: torch.Tensor) -> None:
    if out.dtype != dtype:
        raise ValueError(f"Expected out.dtype == {dtype}, got {out.dtype}")
    if out.shape != A.shape:
        raise ValueError(f"Expected out.shape == {A.shape}, got {out.shape}")
    _dequantize_blockwise_into(A, absmax, code, blocksize, dtype, out)


@kernel("quantize_4bit")
def _quantize_4bit(A: torch.Tensor, blocksize: int, quant_type: str, quant_storage: torch.dtype):
    if blocksize not in _4BIT_BLOCKSIZES:
        raise ValueError(f"invalid blocksize {blocksize}")
    if quant_type not in _QT_ID:
        raise ValueError(f"quant_type must be nf4 or fp4, got {quant_type}")
    sfx = _suffix(A.dtype, "Blockwise 4bit quantization")
    A = A.contiguous()
    n = A.numel()
    _check_sizes("quantize_4bit", n)
    absmax = torch.empty((-(n // -blocksize),), device=A.device, dtype=torch.float32)
    out = torch.empty(((n + 1) // (quant_storage.itemsize * 2), 1), device=A.device, dtype=quant_storage)
    with _on_device(A):
        lib.cbnb_b200_quantize_blockwise(None, A.data_ptr(), absmax.data_ptr(), out.data_ptr(), blocksize, n,
                                         _QT_ID[quant_type], _DTYPE_ID[A.dtype], _stream(A))
    lib.check(f"quantize_4bit[{sfx},{quant_type}]")
    return out, absmax


def _dequantize_4bit_into(A, absmax, blocksize, quant_type, dtype, out) -> None:
    if quant_type not in _QT_ID:
        raise ValueError(f"quant_type must be nf4 or fp4, got {quant_type}")
    sfx = _suffix(dtype, "Blockwise 4bit dequantization")
    A = A.contiguous()
    _check_sizes("dequantize_4bit", out.numel())
    with _on_device(A):
        getattr(lib, f"cdequantize_blockwise_{sfx}_{quant_type}")(None, A.data_ptr(), absmax.data_ptr(),
                                                                  out.data_ptr(), blocksize, out.numel(), _stream(A))
    lib.check(f"dequantize_4bit[{sfx},{quant_type}]")


@kernel("dequantize_4bit")
def _dequantize_4bit(A, absmax, blocksize: int, quant_type: str, shape: Sequence[int], dtype: torch.dtype):
    out = torch.empty(shape, dtype=dtype, device=A.device)
    _dequantize_4bit_into(A, absmax, blocksize, quant_type, dtype, out)
    return out


@kernel("dequantize_4bit.out")
def _dequantize_4bit_out(A, absmax, blocksize: int, quant_type: str, shape: Sequence[int], dtype: torch.dtype,
                         out: torch.Tensor) -> None:
    if out.shape != tuple(shape):
        raise ValueError(f"Expected out.shape == {shape}, got {out.shape}")
    if out.dtype != dtype:
        raise ValueError(f"Expected out.dtype == {dtype}, got {out.dtype}")
    _dequantize_4bit_into(A, absmax, blocksize, quant_type, dtype, out)


# ====================================================================================== 4-bit GEMM
def gemm_4bit_into(A, B, shapeB, absmax, blocksize, quant_type, bias, absmax_8bit, absmax_code, absmax_offset,
                   out: torch.Tensor, ldc: int) -> None:
    """out[:, :N] (row stride ldc) = A . dequant(B)^T + bias.  Shared by the op and the sharded linear."""
    K = A.shape[-1]
    M = A.numel() // K if K else 0
    N = shapeB[0]
    if K != shapeB[1]:
        raise RuntimeError(f"A inner dim ({K}) does not match weight ({shapeB[1]})")
    _check_sizes("gemm_4bit", M, N, K, ldc)
    if absmax.dtype != torch.float32:
        raise RuntimeError(f"absmax must be float32, got {absmax.dtype}")
    if quant_type not in _QT_ID:
        raise RuntimeError(f"quant_type must be nf4 or fp4, got {quant_type}")
    if bias is not None:
        if bias.ndim != 1:
            raise RuntimeError(f"bias must be 1D, got {bias.ndim}D")
        if bias.dtype != A.dtype:
            raise RuntimeError(f"bias dtype ({bias.dtype}) must match A dtype ({A.dtype})")
    if A.dtype not in _DTYPE_ID:
        raise RuntimeError(f"unsupported dtype {A.dtype}")
    if (absmax_8bit is None) != (absmax_code is None) or (absmax_8bit is None) != (absmax_offset is None):
        raise RuntimeError("absmax_8bit, absmax_code and absmax_offset must be given together")
    if blocksize not in _4BIT_BLOCKSIZES:
        raise RuntimeError(f"invalid blocksize {blocksize}")
    A = A.contiguous()
    B = B.contiguous()
    off = None
    if absmax_offset is not None:
        off = absmax_offset.to(dtype=torch.float32).contiguous()
    with _on_device(A):
        lib.cbnb_b200_gemm_4bit_strided(
            A.data_ptr(), B.data_ptr(), absmax.data_ptr(),
            absmax_8bit.data_ptr() if absmax_8bit is not None else None,
            absmax_code.data_ptr() if absmax_code is not None else None,
            off.data_ptr() if off is not None else None,
            out.data_ptr(), bias.data_ptr() if bias is not None else None,
            M, N, K, ldc, blocksize, _QT_ID[quant_type], _DTYPE_ID[A.dtype], _stream(A))
    lib.check("gemm_4bit")


def gemm_4bit_multi_out(A, B, shapeB, absmax, blocksize: int, quant_type: str, bias, absmax_8bit, absmax_code,
                        absmax_offset, out_ptrs, ldc: int) -> bool:
    """Fused GEMM + all-gather: every output element is stored to each raw device address in
    ``out_ptrs`` (local buffer first, then the peers' -- symmetric memory / CUDA IPC mappings), row
    stride ``ldc`` elements.  Returns False when the shape does not take the wgmma kernel (the caller
    falls back to a local output + a collective)."""
    N, K = shapeB
    M = A.numel() // K
    if A.dtype not in (torch.float16, torch.bfloat16):
        return False
    if not 1 <= len(out_ptrs) <= 8:
        raise RuntimeError("gemm_4bit_multi_out: between 1 and 8 destinations")
    A = A.contiguous()
    B = B.contiguous()
    off = absmax_offset.to(dtype=torch.float32).contiguous() if absmax_offset is not None else None
    arr = (ct.c_void_p * len(out_ptrs))(*[int(p) for p in out_ptrs])
    with _on_device(A):
        rc = lib.cbnb_b200_gemm_4bit_multi_out(
            A.data_ptr(), B.data_ptr(), absmax.data_ptr(),
            absmax_8bit.data_ptr() if absmax_8bit is not None else None,
            absmax_code.data_ptr() if absmax_code is not None else None,
            off.data_ptr() if off is not None else None,
            ct.cast(arr, ct.c_void_p), len(out_ptrs), bias.data_ptr() if bias is not None else None,
            M, N, K, ldc, blocksize, _QT_ID[quant_type], _DTYPE_ID[A.dtype], _stream(A))
    lib.check("gemm_4bit_multi_out")
    return rc == 0


@kernel("gemm_4bit")
def _gemm_4bit(A, B, shapeB, absmax, blocksize: int, quant_type: str, bias=None, absmax_8bit=None, absmax_code=None,
               absmax_offset=None):
    N = shapeB[0]
    out = torch.empty((*A.shape[:-1], N), dtype=A.dtype, device=A.device)
    if out.numel() == 0:
        return out
    gemm_4bit_into(A, B, shapeB, absmax, blocksize, quant_type, bias, absmax_8bit, absmax_code, absmax_offset, out, N)
    return out


def _gemv_4bit_into(A, B, shapeB, absmax, code, blocksize, out) -> None:
    if blocksize not in _4BIT_BLOCKSIZES:
        raise ValueError(f"invalid blocksize {blocksize}")
    sfx = _suffix(A.dtype, "gemv_4bit")
    n_out, k = shapeB[0], shapeB[1]
    A = A.contiguous()
    with _on_device(A):
        getattr(lib, f"cgemm_4bit_inference_naive_{sfx}")(n_out, 1, k, A.data_ptr(), B.data_ptr(), absmax.data_ptr(),
                                                          code.data_ptr(), out.data_ptr(), n_out, (k + 1) // 2, n_out,
                                                          blocksize, _stream(A))
    lib.check("gemv_4bit")


@kernel("gemv_4bit")
def _gemv_4bit(A, B, shapeB, absmax, code, blocksize: int):
    out = torch.empty((*A.shape[:-1], shapeB[0]), device=A.device, dtype=A.dtype)
    _gemv_4bit_into(A, B, shapeB, absmax, code, blocksize, out)
    return out


@kernel("gemv_4bit.out")
def _gemv_4bit_out(A, B, shapeB, absmax, code, blocksize: int, out: torch.Tensor) -> None:
    expect = (*A.shape[:-1], shapeB[0])
    if out.shape != expect:
        raise ValueError(f"Expected out.shape == {expect}, got {out.shape}")
    if out.dtype != A.dtype:
        raise ValueError(f"Expected out.dtype == {A.dtype}, got {out.dtype}")
    _gemv_4bit_into(A, B, shapeB, absmax, code, blocksize, out)


# ====================================================================================== LLM.int8()
def _int8_matmul_into(A: torch.Tensor, B: torch.Tensor, out: torch.Tensor):
    """out[..., N] int32 = A[..., K] int8 . B[N, K]^T int8 (exact)."""
    if B.dtype != torch.int8:
        raise ValueError("B must be int8")
    if A.dtype != torch.int8:
        raise ValueError("A must be int8")
    if B.ndim != 2:
        raise ValueError("Only two dimensional matrices are supported for argument B")
    if A.ndim not in (2, 3):
        raise ValueError("Only two or three dimensional matrices are supported for argument A")
    if prod(A.shape) <= 0:
        raise ValueError(f"Input tensor dimensions need to be > 0: {A.shape}")
    if out.dtype != torch.int32:
        raise ValueError(f"out must be int32, got {out.dtype}")
    shape_c = (*A.shape[:-1], B.shape[0])
    if out.shape != shape_c:
        raise ValueError(f"Output shape {out.shape} does not match expected shape {shape_c}")
    N, K = B.shape
    if A.shape[-1] != K:
        raise ValueError(f"int8_linear_matmul only supports B^T @ A. Inner dimensions do not match: "
                         f"B @ A = {tuple(A.shape)} @ {tuple(B.shape)}")
    M = prod(A.shape[:-1])
    A = A.contiguous()
    B = B.contiguous()
    with _on_device(A):
        # reference argument order (column-major view): m = N, n = M, k = K, A = weights, B = activations
        rc = lib.cigemmlt_32(lib.get_context(), N, M, K, B.data_ptr(), A.data_ptr(), out.data_ptr(), None, K, K, N,
                             _stream(A))
    lib.check("int8_linear_matmul")
    if rc == 100:
        # inner dimension not a multiple of 16 bytes (TMA row pitch) or unaligned views: zero-pad K to the next
        # multiple of 16 (zeros add nothing to an integer dot product) and run the same exact kernel.  (The
        # reference's escape hatch for K % 4 != 0 is an fp32 matmul, reference backends/cuda/ops.py:126-128, which
        # is only exact below 2^24.)
        Kp = -(-K // 16) * 16
        Ap = torch.zeros((M, Kp), device=A.device, dtype=torch.int8)
        Bp = torch.zeros((N, Kp), device=A.device, dtype=torch.int8)
        Ap[:, :K] = A.reshape(M, K)
        Bp[:, :K] = B
        with _on_device(A):
            rc = lib.cigemmlt_32(lib.get_context(), N, M, Kp, Bp.data_ptr(), Ap.data_ptr(), out.data_ptr(), None, Kp, Kp,
                                 N, _stream(A))
        lib.check("int8_linear_matmul (padded K)")
    if rc != 0:
        raise RuntimeError(f"int8 GEMM failed (code {rc}): A={tuple(A.shape)} B={tuple(B.shape)}")
    return out


@kernel("int8_linear_matmul")
def _int8_linear_matmul(A: torch.Tensor, B: torch.Tensor):
    out = torch.empty((*A.shape[:-1], B.shape[0]), device=A.device, dtype=torch.int32)
    return _int8_matmul_into(A, B, out)


@kernel("int8_linear_matmul.out")
def _int8_linear_matmul_out(A: torch.Tensor, B: torch.Tensor, out: torch.Tensor) -> None:
    _int8_matmul_into(A, B, out)


@kernel("int8_mm_dequant")
def _int8_mm_dequant(A, row_stats, col_stats, dtype: Optional[torch.dtype] = None, bias: Optional[torch.Tensor] = None):
    if A.dtype != torch.int32:
        raise ValueError(f"A must be int32, got {A.dtype}")
    if row_stats.dtype != torch.float32:
        raise ValueError(f"row_stats must be float32, got {row_stats.dtype}")
    if col_stats.dtype != torch.float32:
        raise ValueError(f"col_stats must be float32, got {col_stats.dtype}")
    A = A.contiguous()
    out = torch.empty_like(A, dtype=torch.float16)
    fused_bias = bias if (bias is not None and bias.dtype == torch.float16) else None
    with _on_device(A):
        lib.cdequant_mm_int32_fp16(A.data_ptr(), row_stats.data_ptr(), col_stats.data_ptr(), out.data_ptr(),
                                   fused_bias.data_ptr() if fused_bias is not None else None,
                                   A.numel() // A.shape[-1], A.shape[-1], _stream(A))
    lib.check("int8_mm_dequant")
    if bias is not None and fused_bias is None:
        out.add_(bias)
    return out.to(dtype or torch.float16)


def int8_vectorwise_quant_flags(A: torch.Tensor, threshold: float):
    """Row quantisation + per-column outlier flags in ONE kernel (fp16 or bf16 input)."""
    if A.dtype not in (torch.float16, torch.bfloat16):
        raise ValueError(f"A must be float16 or bfloat16, got {A.dtype}")
    A = A.contiguous()
    cols = A.shape[-1]
    rows = A.numel() // cols
    row_stats = torch.empty(rows, device=A.device, dtype=torch.float32)
    q = torch.empty(A.shape, device=A.device, dtype=torch.int8)
    flags = torch.zeros(cols, device=A.device, dtype=torch.int32) if threshold > 0.0 else None
    with _on_device(A):
        lib.cbnb_b200_int8_vector_quant_flags(A.data_ptr(), q.data_ptr(), row_stats.data_ptr(),
                                              flags.data_ptr() if flags is not None else None, float(threshold), rows,
                                              cols, _DTYPE_ID[A.dtype], _stream(A))
    lib.check("int8_vectorwise_quant")
    return q, row_stats, flags


@kernel("int8_vectorwise_quant")
def _int8_vectorwise_quant(A: torch.Tensor, threshold=0.0):
    if A.dtype != torch.float16:
        raise ValueError(f"A must be float16, got {A.dtype}")
    if threshold < 0.0:
        raise ValueError("threshold must be non-negative")
    q, row_stats, flags = int8_vectorwise_quant_flags(A, threshold)
    outlier_cols = None
    if flags is not None:
        outlier_cols = torch.nonzero(flags).view(-1)  # data-dependent shape: the one unavoidable sync
        rows = q.numel() // q.shape[-1]
        if outlier_cols.numel() and rows > 1:
            with _on_device(q):
                lib.cbnb_b200_int8_zero_columns(q.data_ptr(), outlier_cols.data_ptr(), int(outlier_cols.numel()), rows,
                                                q.shape[-1], _stream(q))
            lib.check("int8_vectorwise_quant (outlier columns)")
    return q, row_stats, outlier_cols


@kernel("int8_double_quant")
def _int8_double_quant(A: torch.Tensor, threshold=0.0):
    """Row-wise and column-wise int8 codes + statistics (reference backends/cuda/ops.py:257-296).  The column half is one
    native absmax pass and one quantise pass (`csrc/int8.cu`), bit-identical to the reference's five PyTorch kernels
    (`tests/test_gpu_int8.py`); the PyTorch formula below remains for anything the native entry does not take."""
    q_row, row_stats, outlier_cols = torch.ops.bitsandbytes.int8_vectorwise_quant.default(A, threshold=threshold)
    cols = A.shape[-1]
    rows = A.numel() // cols if cols else 0
    if A.dtype == torch.float16 and rows > 0:  # (the row half above accepts fp16 only, as the reference's does)
        _check_sizes("int8_double_quant", A.numel())
        A2 = A.reshape(rows, cols).contiguous()
        q_col = torch.empty((rows, cols), device=A.device, dtype=torch.int8)
        col_stats = torch.empty((cols,), device=A.device, dtype=torch.float32)
        with _on_device(A):
            rc = lib.cbnb_b200_int8_col_quant(A2.data_ptr(), q_col.data_ptr(), col_stats.data_ptr(), float(threshold), rows,
                                              cols, _DTYPE_ID[A.dtype], _stream(A))
        lib.check("int8_double_quant")
        if rc == 0:
            return q_row, q_col.view(A.shape), row_stats, col_stats, outlier_cols
    absA = A.abs().view(-1, A.shape[-1])
    mask = None
    if threshold > 0.0:
        mask = absA >= threshold
        absA = absA.masked_fill(mask, 0.0)
    col_stats = absA.amax(dim=0).float()
    Ac = A.view(-1, A.shape[-1])
    if mask is not None:
        Ac = Ac.masked_fill(mask, 0.0)
    q_col = torch.round(Ac.mul(127.0) / col_stats.unsqueeze(0)).to(torch.int8).view(A.shape)
    return q_row, q_col, row_stats, col_stats.flatten().float(), outlier_cols


def _fused_scaled_mm(CA, CB, SCA, SCB, bias, dtype) -> Optional[torch.Tensor]:
    """int8 GEMM with the dequant epilogue in-kernel; None if the shape is not supported."""
    if dtype not in (torch.float16, torch.bfloat16):
        return None
    N, K = CB.shape
    M = CA.numel() // K
    if K % 16 != 0 or M == 0:
        return None
    if bias is not None and bias.dtype != dtype:
        return None  # keep the reference's rounding order for mixed-dtype biases (unfused chain below)
    CA = CA.contiguous()
    CB = CB.contiguous()
    out = torch.empty((*CA.shape[:-1], N), device=CA.device, dtype=dtype)
    with _on_device(CA):
        rc = lib.cbnb_b200_int8_scaled_mm(CA.data_ptr(), CB.data_ptr(), SCA.data_ptr(), SCB.data_ptr(),
                                          bias.data_ptr() if bias is not None else None, out.data_ptr(), M, N, K,
                                          _DTYPE_ID[dtype], _stream(CA))
    lib.check("int8_scaled_mm")
    return out if rc == 0 else None


@kernel("int8_scaled_mm")
def _int8_scaled_mm(A, B, row_stats, col_stats, bias=None, dtype=None):
    dtype = dtype or torch.float16
    if row_stats.dtype == torch.float32 and col_stats.dtype == torch.float32 and A.dtype == torch.int8:
        out = _fused_scaled_mm(A, B, row_stats.contiguous(), col_stats.contiguous(), bias, dtype)
        if out is not None:
            return out
    acc = torch.ops.bitsandbytes.int8_linear_matmul.default(A, B)
    return torch.ops.bitsandbytes.int8_mm_dequant.default(acc, row_stats, col_stats, dtype=dtype, bias=bias)


def _fused_mixed_mm(A, CA, CB, SCA, SCB, outlier_cols, bias):
    """The whole LLM.int8() decomposition in two launches: one gathers subA and dequantises the outlier weight
    columns into [N, jpad], the other is the int8 wgmma GEMM whose epilogue adds the outlier term.
    Returns (out, subA) or None when the shape is not served (K % 16, > 64 outlier columns, dtype)."""
    dtype = A.dtype
    if dtype not in (torch.float16, torch.bfloat16) or CA.dtype != torch.int8 or CB.dtype != torch.int8:
        return None
    if SCA.dtype != torch.float32 or SCB.dtype != torch.float32:
        return None
    if bias is not None and bias.dtype != dtype:
        return None
    N, K = CB.shape
    M = CA.numel() // K
    J = int(outlier_cols.numel())
    if K % 16 != 0 or M == 0 or J == 0 or J > 64:
        return None
    jpad = -(-J // 8) * 8
    A2 = A.reshape(-1, K).contiguous()
    CA = CA.contiguous()
    CB = CB.contiguous()
    SCA = SCA.contiguous()
    SCB = SCB.contiguous()
    cols = outlier_cols.to(torch.int64).contiguous()
    subA_pad = torch.empty((M, jpad), device=A.device, dtype=dtype)
    subBT = torch.empty((N, jpad), device=A.device, dtype=dtype)
    out = torch.empty((*CA.shape[:-1], N), device=A.device, dtype=dtype)
    with _on_device(A):
        lib.cbnb_b200_int8_outlier_prep(A2.data_ptr(), CB.data_ptr(), SCB.data_ptr(), cols.data_ptr(), J, jpad, M, N, K,
                                        _DTYPE_ID[dtype], subA_pad.data_ptr(), subBT.data_ptr(), _stream(A))
        rc = lib.cbnb_b200_int8_mixed_mm(CA.data_ptr(), CB.data_ptr(), SCA.data_ptr(), SCB.data_ptr(),
                                         bias.data_ptr() if bias is not None else None, subA_pad.data_ptr(),
                                         subBT.data_ptr(), jpad, out.data_ptr(), M, N, K, _DTYPE_ID[dtype], _stream(A))
    lib.check("int8_mixed_scaled_mm")
    if rc != 0:
        return None
    subA = subA_pad[:, :J].reshape(*A.shape[:-1], J)
    return out, (subA if jpad == J else subA.contiguous())


@kernel("int8_mixed_scaled_mm")
def _int8_mixed_scaled_mm(A, CA, CB, SCA, SCB, outlier_cols=None, bias=None):
    """LLM.int8() forward: int8 part + the fp16/bf16 outlier columns (reference default/ops.py:64-100)."""
    if outlier_cols is not None and outlier_cols.numel():
        fused = _fused_mixed_mm(A, CA, CB, SCA, SCB, outlier_cols, bias)
        if fused is not None:
            return fused
        # shapes the fused kernel does not take (> 64 outlier columns, K % 16 != 0): the reference's own chain
        subA = A[..., outlier_cols].contiguous()
        # reference _ops.py:118-121: CB * SCB * (1/127) in fp32, then to A.dtype
        subB = torch.ops.bitsandbytes.int8_vectorwise_dequant.default(CB[:, outlier_cols].contiguous(), SCB)
        subB = subB.to(A.dtype).t()
        out = torch.ops.bitsandbytes.int8_scaled_mm.default(CA, CB, SCA, SCB, bias=bias, dtype=A.dtype)
        out = out.view(-1, out.shape[-1]).addmm(subA.view(-1, subA.shape[-1]), subB).view(out.shape)
        return out, subA
    subA = torch.empty(0, device=A.device, dtype=A.dtype)  # keeps torch.compile's output arity fixed
    out = torch.ops.bitsandbytes.int8_scaled_mm.default(CA, CB, SCA, SCB, bias=bias, dtype=A.dtype)
    return out, subA


# ------------------------------------------------------------------------------------------ optimizers (section 8 f-4)
# optimizer name -> (native id, bf16 served by the reference-named 32-bit symbol)  (reference
# backends/cuda/ops.py:985-1066: lamb is adam with max_unorm, lars is momentum with max_unorm)
_OPTIMIZER_ID = {"adam": 0, "lamb": 0, "momentum": 1, "lars": 1, "rmsprop": 2, "adagrad": 3, "lion": 4, "ademamix": 5}
_OPTIMIZER_8BIT = ("adam", "momentum", "rmsprop", "adagrad", "lion", "ademamix")


def _optional_ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


@kernel("optimizer_update_32bit")
def _optimizer_update_32bit(optimizer_name, g, p, state1, state2, unorm_vec, max_unorm, param_norm, beta1, beta2, beta3,
                            alpha, eps, weight_decay, step, lr, gnorm_scale, skip_zeros=False):
    """One in-place step with fp32 state (reference backends/cuda/ops.py:1069-1123, kernels csrc/kernels.cu:531-909)."""
    if optimizer_name not in _OPTIMIZER_ID:
        raise ValueError(f"Unsupported optimizer name: {optimizer_name}. Supported optimizers: {list(_OPTIMIZER_ID)}")
    if g.dtype not in _DTYPE_ID:
        raise ValueError(f"Gradient+optimizer bit data type combination not supported: grad {g.dtype}, optimizer {state1.dtype}")
    if g.dtype != p.dtype or g.numel() != p.numel():
        raise ValueError("optimizer_update_32bit: g and p must have the same dtype and number of elements")
    for t in (g, p, state1, state2, unorm_vec):
        if t is not None and not t.is_contiguous():
            raise ValueError("optimizer_update_32bit: tensors must be contiguous")
    with _on_device(g):
        rc = lib.cbnb_b200_optimizer_update_32bit(_OPTIMIZER_ID[optimizer_name], _DTYPE_ID[g.dtype], g.data_ptr(),
                                                  p.data_ptr(), state1.data_ptr(), _optional_ptr(state2),
                                                  _optional_ptr(unorm_vec), float(max_unorm), float(param_norm),
                                                  float(beta1), float(beta2), float(beta3), float(alpha), float(eps),
                                                  float(weight_decay), int(step), float(lr), float(gnorm_scale),
                                                  bool(skip_zeros), g.numel(), _stream(g))
    lib.check("optimizer_update_32bit")
    if rc != 0:
        raise RuntimeError(f"optimizer_update_32bit: native call returned {rc}")


@kernel("optimizer_update_8bit_blockwise")
def _optimizer_update_8bit_blockwise(optimizer_name, g, p, state1, state2, beta1, beta2, beta3, alpha, eps, step, lr, qmap1,
                                     qmap2, absmax1, absmax2, weight_decay, gnorm_scale, skip_zeros=False):
    """One in-place step with blockwise (256) 8-bit state (reference backends/cuda/ops.py:1126-1209, kernels
    csrc/kernels.cu:914-1325)."""
    if optimizer_name not in _OPTIMIZER_8BIT:
        raise ValueError(f"Unsupported optimizer name: {optimizer_name}. Supported optimizers: {list(_OPTIMIZER_8BIT)}")
    if g.dtype not in _DTYPE_ID:
        raise ValueError(f"Unsupported gradient dtype: {g.dtype}. Supported dtypes: torch.float32, torch.float16, torch.bfloat16")
    if g.dtype != p.dtype or g.numel() != p.numel():
        raise ValueError("optimizer_update_8bit_blockwise: g and p must have the same dtype and number of elements")
    two = optimizer_name in ("adam", "ademamix")
    if two and (state2 is None or qmap2 is None or absmax2 is None):
        raise ValueError(f"optimizer_update_8bit_blockwise: {optimizer_name} needs state2, qmap2 and absmax2")
    for t in (g, p, state1, state2, qmap1, qmap2, absmax1, absmax2):
        if t is not None and not t.is_contiguous():
            raise ValueError("optimizer_update_8bit_blockwise: tensors must be contiguous")
    with _on_device(g):
        rc = lib.cbnb_b200_optimizer_update_8bit_blockwise(
            _OPTIMIZER_ID[optimizer_name], _DTYPE_ID[g.dtype], p.data_ptr(), g.data_ptr(), state1.data_ptr(),
            _optional_ptr(state2), float(beta1), float(beta2), float(beta3), float(alpha), float(eps), int(step), float(lr),
            qmap1.data_ptr(), _optional_ptr(qmap2), absmax1.data_ptr(), _optional_ptr(absmax2), float(weight_decay),
            float(gnorm_scale), bool(skip_zeros), g.numel(), _stream(g))
    lib.check("optimizer_update_8bit_blockwise")
    if rc != 0:
        raise RuntimeError(f"optimizer_update_8bit_blockwise: native call returned {rc}")
