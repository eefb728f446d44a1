"""Host side of the sm_90a kernels: argument checking, output allocation, the ctypes call.

Plays the role of the reference's ``bitsandbytes/backends/cuda/ops.py`` (:78-982) for the
hot path, with three structural differences:

* no per-architecture heuristic (reference :583-811) and no dequantize + cuBLAS fallback
  (:904-916): ``gemm_4bit`` always runs a fused kernel -- wgmma for 16-bit activations and,
  when PyTorch allows TF32 for fp32 matmuls, for fp32 ones on TF32 tensor cores; CUDA cores
  for other fp32 calls / odd shapes; the choice is made inside the library;
* ``int8_vectorwise_quant`` finds outlier columns inside the quantisation kernel instead
  of three torch kernels and a host sync (reference :230-236); the data-dependent
  ``outlier_cols`` tensor still has to be materialised (``nonzero``), once, except on the
  CUDA-graph route ``int8_mixed_mm_flags``, which keeps the columns and their count on the device;
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

from .._ops import MAX_EXPERTS, check_grouped, check_int8_grouped, kernel
from .. import cextension as cext
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
_DTYPE_ID_TF32 = 3  # fp32 activations with TF32 allowed: the library's TF32 tensor-core route


def gemm_4bit_dtype_id(dtype: torch.dtype) -> int:
    """The native dtype id of a 4-bit GEMM with activations of ``dtype``.  fp32 follows PyTorch's fp32 matmul
    precision, as cuBLAS does for ``torch.matmul``: 3 (TF32 allowed) when
    ``torch.backends.cuda.matmul.fp32_precision`` is ``"tf32"`` -- set directly, inherited from
    ``torch.backends.fp32_precision``, or through ``allow_tf32 = True`` / ``set_float32_matmul_precision("high")`` or
    ``("medium")`` -- and 0 (fp32 CUDA-core products) otherwise.  The setting is read on every call, so a CUDA graph
    keeps the route in force when it was captured.  (Only ``fp32_precision`` is read: the legacy getters raise once
    the legacy and the per-backend APIs have been mixed.)"""
    if dtype == torch.float32 and torch.backends.cuda.matmul.fp32_precision == "tf32":
        return _DTYPE_ID_TF32
    return _DTYPE_ID[dtype]


def _gemm_4bit_operands(what: str, A, B, shapeB, absmax, blocksize, quant_type, bias, absmax_8bit, absmax_code,
                        absmax_offset, ldc: int):
    """The checked operands of a 4-bit GEMM: (contiguous A, contiguous B, the fp32 offset or None, M, N, K)."""
    N, K = shapeB[0], shapeB[1]
    if A.shape[-1] != K:
        raise RuntimeError(f"A inner dim ({A.shape[-1]}) does not match weight ({K})")
    M = A.numel() // K if K else 0
    _check_sizes(what, M, N, K, ldc)
    if A.dtype not in _DTYPE_ID:
        raise RuntimeError(f"unsupported dtype {A.dtype}")
    off = _weight_operands(absmax, blocksize, quant_type, absmax_8bit, absmax_code, absmax_offset)
    if bias is not None:
        if bias.ndim != 1:
            raise RuntimeError(f"bias must be 1D, got {bias.ndim}D")
        if bias.dtype != A.dtype:
            raise RuntimeError(f"bias dtype ({bias.dtype}) must match A dtype ({A.dtype})")
    return A.contiguous(), B.contiguous(), off, M, N, K


def _weight_operands(absmax, blocksize, quant_type, absmax_8bit, absmax_code, absmax_offset):
    """Checks the statistics of a packed 4-bit weight; returns the fp32 offset of nested statistics, or None."""
    if absmax.dtype != torch.float32:
        raise RuntimeError(f"absmax must be float32, got {absmax.dtype}")
    if quant_type not in _QT_ID:
        raise RuntimeError(f"quant_type must be nf4 or fp4, got {quant_type}")
    if blocksize not in _4BIT_BLOCKSIZES:
        raise RuntimeError(f"invalid blocksize {blocksize}")
    if (absmax_8bit is None) != (absmax_code is None) or (absmax_8bit is None) != (absmax_offset is None):
        raise RuntimeError("absmax_8bit, absmax_code and absmax_offset must be given together")
    return absmax_offset.to(dtype=torch.float32).contiguous() if absmax_offset is not None else None


def gemm_4bit_into(A, B, shapeB, absmax, blocksize, quant_type, bias, absmax_8bit, absmax_code, absmax_offset,
                   out: torch.Tensor, ldc: int) -> None:
    """out[:, :N] (row stride ldc) = A . dequant(B)^T + bias.  Shared by the op and the sharded linear.  fp32 ``A``
    runs on TF32 tensor cores when PyTorch's fp32 matmul precision allows TF32 (:func:`gemm_4bit_dtype_id`)."""
    A, B, off, M, N, K = _gemm_4bit_operands("gemm_4bit", A, B, shapeB, absmax, blocksize, quant_type, bias,
                                             absmax_8bit, absmax_code, absmax_offset, ldc)
    with _on_device(A):
        lib.cbnb_b200_gemm_4bit_strided(
            A.data_ptr(), B.data_ptr(), absmax.data_ptr(),
            absmax_8bit.data_ptr() if absmax_8bit is not None else None,
            absmax_code.data_ptr() if absmax_code is not None else None,
            off.data_ptr() if off is not None else None,
            out.data_ptr(), bias.data_ptr() if bias is not None else None,
            M, N, K, ldc, blocksize, _QT_ID[quant_type], gemm_4bit_dtype_id(A.dtype), _stream(A))
    lib.check("gemm_4bit")


def gemm_4bit_multi_out(A, B, shapeB, absmax, blocksize: int, quant_type: str, bias, absmax_8bit, absmax_code,
                        absmax_offset, out_ptrs, ldc: int) -> bool:
    """Fused GEMM + all-gather: every output element is stored to each destination in ``out_ptrs`` (local buffer
    first, then the peers' -- symmetric memory / CUDA IPC mappings), row stride ``ldc`` elements.  A destination is a
    tensor of A's dtype, checked here, or a raw device address, which the caller vouches for.  Returns False when the
    shape does not take the wgmma kernel (the caller falls back to a local output + a collective)."""
    A, B, off, M, N, K = _gemm_4bit_operands("gemm_4bit_multi_out", A, B, shapeB, absmax, blocksize, quant_type, bias,
                                             absmax_8bit, absmax_code, absmax_offset, ldc)
    ptrs = _dest_ptrs("gemm_4bit_multi_out", out_ptrs, A.dtype, A.device, M, N, ldc, RuntimeError)
    if A.dtype not in (torch.float16, torch.bfloat16):
        return False
    arr = (ct.c_void_p * len(ptrs))(*ptrs)
    with _on_device(A):
        rc = lib.cbnb_b200_gemm_4bit_multi_out(
            A.data_ptr(), B.data_ptr(), absmax.data_ptr(),
            absmax_8bit.data_ptr() if absmax_8bit is not None else None,
            absmax_code.data_ptr() if absmax_code is not None else None,
            off.data_ptr() if off is not None else None,
            ct.cast(arr, ct.c_void_p), len(ptrs), bias.data_ptr() if bias is not None else None,
            M, N, K, ldc, blocksize, _QT_ID[quant_type], _DTYPE_ID[A.dtype], _stream(A))
    lib.check("gemm_4bit_multi_out")
    return rc == 0


def gemm_4bit_partial(A, B, shapeB, absmax, blocksize: int, quant_type: str, absmax_8bit, absmax_code, absmax_offset,
                      outs, ldc: int) -> bool:
    """Partial GEMM of a row-sharded layer: ``P[m, n] = sum_k A[m, k] * dequant(B)[n, k]`` in fp32, with no bias and no
    rounding, stored to every destination in ``outs`` at row stride ``ldc`` (elements).  A destination is an fp32
    CUDA tensor, checked here, or a raw device address (a peer's symmetric-memory slot), which the caller vouches
    for.  The kernel and its K split are the ones the plain GEMM takes for this shape (fp32 ``A`` follows
    :func:`gemm_4bit_dtype_id`), so with one shard the result is the plain GEMM's accumulator.  Returns False when
    the library does not serve the call (the caller takes another route)."""
    A, B, off, M, N, K = _gemm_4bit_operands("gemm_4bit_partial", A, B, shapeB, absmax, blocksize, quant_type, None,
                                             absmax_8bit, absmax_code, absmax_offset, ldc)
    ptrs = _dest_ptrs("gemm_4bit_partial", outs, torch.float32, A.device, M, N, ldc, RuntimeError)
    if M == 0 or N == 0:
        return True
    arr = (ct.c_void_p * len(ptrs))(*ptrs)
    with _on_device(A):
        rc = lib.cbnb_b200_gemm_4bit_partial(
            A.data_ptr(), B.data_ptr(), absmax.data_ptr(),
            absmax_8bit.data_ptr() if absmax_8bit is not None else None,
            absmax_code.data_ptr() if absmax_code is not None else None,
            off.data_ptr() if off is not None else None,
            ct.cast(arr, ct.c_void_p), len(ptrs), M, N, K, ldc, blocksize, _QT_ID[quant_type],
            gemm_4bit_dtype_id(A.dtype), _stream(A))
    lib.check("gemm_4bit_partial")
    return rc == 0


def gemm_4bit_partial_scatter(A, B, shapeB, absmax, blocksize: int, quant_type: str, absmax_8bit, absmax_code,
                              absmax_offset, outs, ldc: int) -> bool:
    """:func:`gemm_4bit_partial` with the rows scattered over ``outs`` in rank order instead of copied to each: with
    ``w = len(outs)`` and ``M`` rows, row ``m`` is stored to ``outs[m // (M/w)]`` at row ``m % (M/w)`` (row stride
    ``ldc``), the partial of a sequence-parallel layer whose rank s owns tokens ``[s*M/w, (s+1)*M/w)``.  Same kernel,
    K split and fp32 sums as :func:`gemm_4bit_partial`.  ``M % w == 0`` is required."""
    A, B, off, M, N, K = _gemm_4bit_operands("gemm_4bit_partial_scatter", A, B, shapeB, absmax, blocksize, quant_type,
                                             None, absmax_8bit, absmax_code, absmax_offset, ldc)
    n = len(outs)
    if n < 1 or M < n or M % n != 0:
        raise RuntimeError(f"gemm_4bit_partial_scatter: {M} rows do not split evenly over {n} destinations")
    ptrs = _dest_ptrs("gemm_4bit_partial_scatter", outs, torch.float32, A.device, M // n, N, ldc, RuntimeError)
    if N == 0:
        return True
    arr = (ct.c_void_p * n)(*ptrs)
    with _on_device(A):
        rc = lib.cbnb_b200_gemm_4bit_partial_scatter(
            A.data_ptr(), B.data_ptr(), absmax.data_ptr(),
            absmax_8bit.data_ptr() if absmax_8bit is not None else None,
            absmax_code.data_ptr() if absmax_code is not None else None,
            off.data_ptr() if off is not None else None,
            ct.cast(arr, ct.c_void_p), n, M // n, M, N, K, ldc, blocksize, _QT_ID[quant_type],
            gemm_4bit_dtype_id(A.dtype), _stream(A))
    lib.check("gemm_4bit_partial_scatter")
    return rc == 0


def reduce_partials(parts: torch.Tensor, dtype: torch.dtype, bias: Optional[torch.Tensor] = None,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out = dtype((((parts[0] + parts[1]) + ...) + parts[w-1]) + bias)``: the ``[w, M, N]`` fp32 partials of a
    row-sharded layer summed in rank order in fp32, the bias added in fp32, one rounding.  ``out`` may be a
    ``[M, N]`` view with unit column stride and any row stride (a column slice of a wider buffer)."""
    if parts.dtype != torch.float32 or parts.dim() != 3 or not parts.is_cuda:
        raise RuntimeError(f"reduce_partials: parts must be a [world, M, N] float32 CUDA tensor, got {parts.dtype} "
                           f"{tuple(parts.shape)} on {parts.device}")
    if dtype not in _DTYPE_ID:
        raise RuntimeError(f"reduce_partials: unsupported dtype {dtype}")
    world, M, N = parts.shape
    if world < 1:
        raise RuntimeError("reduce_partials: no partials")
    parts = parts.contiguous()
    if bias is not None and (bias.dtype != dtype or bias.shape != (N,) or bias.device != parts.device):
        raise RuntimeError(f"reduce_partials: bias must be {dtype} [{N}] on {parts.device}")
    if bias is not None:
        bias = bias.contiguous()
    if out is None:
        out = torch.empty((M, N), dtype=dtype, device=parts.device)
    elif (out.dtype != dtype or out.shape != (M, N) or out.device != parts.device
          or (M > 1 and out.stride(1) != 1) or out.stride(0) < N):
        raise RuntimeError(f"reduce_partials: out must be {dtype} [{M}, {N}] with unit column stride on {parts.device}")
    _check_sizes("reduce_partials", M, N, out.stride(0), world)
    if M == 0 or N == 0:
        return out
    with _on_device(parts):
        rc = lib.cbnb_b200_reduce_partials(parts.data_ptr(), world, M * N, out.data_ptr(),
                                           bias.data_ptr() if bias is not None else None, M, N, out.stride(0),
                                           _DTYPE_ID[dtype], _stream(parts))
    lib.check("reduce_partials")
    if rc != 0:
        raise RuntimeError(f"reduce_partials: the library refused the call (code {rc})")
    return out


def reduce_partials_ptrs(ptrs, M: int, N: int, dtype: torch.dtype, row0: int = 0, rows: Optional[int] = None,
                         bias: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """:func:`reduce_partials` over 1..8 ``[M, N]`` fp32 partials in separate buffers, listed in rank order, and only
    over the rows ``[row0, row0 + rows)``: ``out[m] = dtype(((ptrs[0] + ptrs[1]) + ...)[row0 + m] + bias)``, the same
    bits as :func:`reduce_partials` on the stacked partials.  A partial is a contiguous fp32 ``[M, N]`` CUDA tensor,
    checked here, or a raw device address (a peer's symmetric-memory slot), which the caller vouches for.  ``out`` may
    be a ``[rows, N]`` view with unit column stride and any row stride."""
    if dtype not in _DTYPE_ID:
        raise RuntimeError(f"reduce_partials_ptrs: unsupported dtype {dtype}")
    rows = M - row0 if rows is None else rows
    if M < 0 or N < 0 or row0 < 0 or rows < 0 or row0 + rows > M:
        raise RuntimeError(f"reduce_partials_ptrs: the row window [{row0}, {row0 + rows}) is outside the {M} rows")
    tensors = [p for p in ptrs if isinstance(p, torch.Tensor)]
    device = out.device if out is not None else tensors[0].device if tensors else torch.device(
        "cuda", torch.cuda.current_device())
    if device.type != "cuda":
        raise RuntimeError(f"reduce_partials_ptrs: the partials must be on a CUDA device, got {device}")
    if any(p.shape != (M, N) or not p.is_contiguous() for p in tensors):
        raise RuntimeError(f"reduce_partials_ptrs: partials must be contiguous [{M}, {N}] tensors (the kernel reads them "
                           "at row stride N)")
    addrs = _dest_ptrs("reduce_partials_ptrs", ptrs, torch.float32, device, M, N, N, RuntimeError)
    if bias is not None and (bias.dtype != dtype or bias.shape != (N,) or bias.device != device):
        raise RuntimeError(f"reduce_partials_ptrs: bias must be {dtype} [{N}] on {device}")
    if bias is not None:
        bias = bias.contiguous()
    if out is None:
        out = torch.empty((rows, N), dtype=dtype, device=device)
    elif (out.dtype != dtype or out.shape != (rows, N) or (N > 1 and out.stride(1) != 1)
          or (rows > 1 and out.stride(0) < N)):
        raise RuntimeError(f"reduce_partials_ptrs: out must be {dtype} [{rows}, {N}] with unit column stride on "
                           f"{device}")
    _check_sizes("reduce_partials_ptrs", M, N, out.stride(0))
    if rows == 0 or N == 0:
        return out
    arr = (ct.c_void_p * len(addrs))(*addrs)
    with _on_device(out):
        rc = lib.cbnb_b200_reduce_partials_ptrs(ct.cast(arr, ct.c_void_p), len(addrs), row0, rows, out.data_ptr(),
                                                bias.data_ptr() if bias is not None else None, M, N, out.stride(0),
                                                _DTYPE_ID[dtype], _stream(out))
    lib.check("reduce_partials_ptrs")
    if rc != 0:
        raise RuntimeError(f"reduce_partials_ptrs: the library refused the call (code {rc})")
    return out


@kernel("gemm_4bit")
def _gemm_4bit(A, B, shapeB, absmax, blocksize: int, quant_type: str, bias=None, absmax_8bit=None, absmax_code=None,
               absmax_offset=None):
    N = shapeB[0]
    out = torch.empty((*A.shape[:-1], N), dtype=A.dtype, device=A.device)
    if out.numel() == 0:
        return out
    gemm_4bit_into(A, B, shapeB, absmax, blocksize, quant_type, bias, absmax_8bit, absmax_code, absmax_offset, out, N)
    return out


@kernel("gemm_4bit_grouped")
def _gemm_4bit_grouped(A, B, shapeB, absmax, blocksize: int, quant_type: str, offs, bias=None, absmax_8bit=None,
                       absmax_code=None, absmax_offset=None):
    """Every expert of a mixture-of-experts layer in one launch: ``out[m] = A[m] . W[e]^T + bias[e]`` for the rows of
    expert e, ``offs[e-1] <= m < offs[e]`` (offs clamped on the device), and 0 for the rows past ``offs[E-1]``.  Nothing
    is read back to the host, so the call can be captured in a CUDA graph."""
    E, N, K = check_grouped(A, B, shapeB, absmax, blocksize, quant_type, offs, bias, absmax_8bit, absmax_code,
                            absmax_offset)
    out = torch.empty((A.shape[0], N), dtype=A.dtype, device=A.device)
    _grouped_launch(A, B, E, N, K, absmax, blocksize, quant_type, offs, bias, absmax_8bit, absmax_code, absmax_offset,
                    out, N)
    return out


def _grouped_out(what: str, out: torch.Tensor, dtype: torch.dtype, device, M: int, N: int, ldc: int) -> None:
    """``out`` is an ``[M, N]`` tensor of ``dtype`` on ``device``, row-major at row stride ``ldc``, with room for it."""
    if (out.dim() != 2 or tuple(out.shape) != (M, N) or (N > 1 and out.stride(1) != 1)
            or (M > 1 and out.stride(0) != ldc)):
        raise RuntimeError(f"{what}: out must be [{M}, {N}] with unit column stride and row stride ldc = {ldc}, got "
                           f"{list(out.shape)} with strides {list(out.stride())}")
    _dest_ptrs(what, [out], dtype, device, M, N, ldc, RuntimeError)


def gemm_4bit_grouped_into(A, B, shapeB, absmax, blocksize: int, quant_type: str, offs, bias, absmax_8bit, absmax_code,
                           absmax_offset, out: torch.Tensor, ldc: int) -> None:
    """The grouped GEMM of ``gemm_4bit_grouped`` into the caller's ``out``, an ``[M, N]`` view at row stride ``ldc``
    (elements) -- a column slice of a wider buffer, as the column-parallel expert layer gathers."""
    E, N, K = check_grouped(A, B, shapeB, absmax, blocksize, quant_type, offs, bias, absmax_8bit, absmax_code,
                            absmax_offset)
    _grouped_out("gemm_4bit_grouped", out, A.dtype, A.device, A.shape[0], N, ldc)
    _grouped_launch(A, B, E, N, K, absmax, blocksize, quant_type, offs, bias, absmax_8bit, absmax_code, absmax_offset,
                    out, ldc)


def _grouped_launch(A, B, E, N, K, absmax, blocksize, quant_type, offs, bias, absmax_8bit, absmax_code, absmax_offset,
                    out, ldc: int) -> None:
    """The native grouped GEMM on operands ``check_grouped`` has accepted, into ``out`` at row stride ``ldc``."""
    M = A.shape[0]
    _check_sizes("gemm_4bit_grouped", M, E * N, K, ldc)
    if M == 0:
        return
    off = _weight_operands(absmax, blocksize, quant_type, absmax_8bit, absmax_code, absmax_offset)
    A, B, offs = A.contiguous(), B.contiguous(), offs.contiguous()
    bias = bias.contiguous() if bias is not None else None
    with _on_device(A):
        rc = lib.cbnb_b200_gemm_4bit_grouped(
            A.data_ptr(), B.data_ptr(), absmax.data_ptr(),
            absmax_8bit.data_ptr() if absmax_8bit is not None else None,
            absmax_code.data_ptr() if absmax_code is not None else None,
            off.data_ptr() if off is not None else None,
            offs.data_ptr(), E, out.data_ptr(), bias.data_ptr() if bias is not None else None,
            M, N, K, ldc, blocksize, _QT_ID[quant_type], _DTYPE_ID[A.dtype], _stream(A))
    lib.check("gemm_4bit_grouped")
    if rc != 0:
        raise RuntimeError(f"gemm_4bit_grouped: the library does not serve this call (code {rc})")


def gemm_4bit_grouped_partial(A, B, shapeB, absmax, blocksize: int, quant_type: str, offs, out: torch.Tensor,
                              ldc: int, mt: int = 0) -> None:
    """The grouped fp32 partial of a row-sharded expert layer: ``out[m, n] = A[m] . dequant(W[e])[n]`` summed in fp32,
    with no bias and no rounding, for the rows of expert e (``offs`` as in ``gemm_4bit_grouped``, clamped on the
    device), and 0 for the rows past ``offs[E-1]``; ``out`` is fp32 at row stride ``ldc``.  The statistics are plain
    fp32 absmax (:func:`~bitsandbytes_b200.parallel.slice_quantized_weight_k` makes them so).  ``mt`` is the token
    tile (16, 32, 64 or 128), 0 for the grouped GEMM's rule, which depends on M and E only: a shard then runs the
    unsharded layer's tile.  Nothing is read back to the host."""
    E, N, K = check_grouped(A, B, shapeB, absmax, blocksize, quant_type, offs)
    M = A.shape[0]
    _check_sizes("gemm_4bit_grouped_partial", M, E * N, K, ldc)
    _grouped_out("gemm_4bit_grouped_partial", out, torch.float32, A.device, M, N, ldc)
    if mt not in (0, 16, 32, 64, 128):
        raise RuntimeError(f"gemm_4bit_grouped_partial: mt must be 0, 16, 32, 64 or 128, got {mt}")
    if M == 0:
        return
    A, B, offs = A.contiguous(), B.contiguous(), offs.contiguous()
    with _on_device(A):
        rc = lib.cbnb_b200_gemm_4bit_grouped_partial(
            A.data_ptr(), B.data_ptr(), absmax.data_ptr(), offs.data_ptr(), E, out.data_ptr(), M, N, K, ldc,
            blocksize, _QT_ID[quant_type], _DTYPE_ID[A.dtype], mt, _stream(A))
    lib.check("gemm_4bit_grouped_partial")
    if rc != 0:
        raise RuntimeError(f"gemm_4bit_grouped_partial: the library does not serve this call (code {rc})")


def reduce_partials_grouped(parts: torch.Tensor, offs: torch.Tensor, dtype: torch.dtype,
                            bias: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """:func:`reduce_partials` for a row-sharded expert layer: ``out[m] = dtype((((parts[0] + parts[1]) + ...) +
    parts[w-1])[m] + bias[e])`` for the rows of expert e, ``offs`` the int32 ``[E]`` end rows (clamped on the device as
    the grouped GEMM clamps them, never read on the host), and 0 for the rows past ``offs[E-1]``.  ``bias`` is
    ``[E, N]``; ``out`` may be an ``[M, N]`` view with unit column stride and any row stride."""
    if parts.dtype != torch.float32 or parts.dim() != 3:
        raise RuntimeError(f"reduce_partials_grouped: parts must be a [world, M, N] float32 tensor, got {parts.dtype} "
                           f"{tuple(parts.shape)}")
    if dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError(f"reduce_partials_grouped: dtype must be float16 or bfloat16, got {dtype}")
    world, M, N = parts.shape
    if world < 1:
        raise RuntimeError("reduce_partials_grouped: no partials")
    if offs.dtype != torch.int32 or offs.dim() != 1 or not 1 <= offs.numel() <= MAX_EXPERTS or offs.device != parts.device:
        raise RuntimeError(f"reduce_partials_grouped: offs must be int32 [E], 1 <= E <= {MAX_EXPERTS}, on "
                           f"{parts.device}, got {offs.dtype} {tuple(offs.shape)} on {offs.device}")
    E = offs.numel()
    if bias is not None and (bias.dtype != dtype or tuple(bias.shape) != (E, N) or bias.device != parts.device):
        raise RuntimeError(f"reduce_partials_grouped: bias must be {dtype} [{E}, {N}] on {parts.device}")
    if out is not None and (out.dtype != dtype or out.shape != (M, N) or out.device != parts.device
                            or (N > 1 and out.stride(1) != 1) or (M > 1 and out.stride(0) < N)):
        raise RuntimeError(f"reduce_partials_grouped: out must be {dtype} [{M}, {N}] with unit column stride on "
                           f"{parts.device}")
    if not parts.is_cuda:
        raise RuntimeError(f"reduce_partials_grouped: the partials must be on a CUDA device, got {parts.device}")
    parts, offs = parts.contiguous(), offs.contiguous()
    bias = bias.contiguous() if bias is not None else None
    if out is None:
        out = torch.empty((M, N), dtype=dtype, device=parts.device)
    _check_sizes("reduce_partials_grouped", M, E * N, out.stride(0), world)
    if M == 0 or N == 0:
        return out
    with _on_device(parts):
        rc = lib.cbnb_b200_reduce_partials_grouped(parts.data_ptr(), world, M * N, offs.data_ptr(), E, out.data_ptr(),
                                                   bias.data_ptr() if bias is not None else None, M, N, out.stride(0),
                                                   _DTYPE_ID[dtype], _stream(parts))
    lib.check("reduce_partials_grouped")
    if rc != 0:
        raise RuntimeError(f"reduce_partials_grouped: the library refused the call (code {rc})")
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


def int8_zero_columns(q: torch.Tensor, cols: torch.Tensor) -> None:
    """q[..., cols] = 0 in place, for contiguous int8 codes and int64 column indices on q's device."""
    if q.dtype != torch.int8 or not q.is_contiguous():
        raise ValueError("q must be contiguous int8")
    if cols.dtype != torch.int64 or not cols.is_contiguous():
        raise ValueError("cols must be contiguous int64")
    rows = q.numel() // q.shape[-1]
    _check_sizes("int8_zero_columns", rows, q.shape[-1], cols.numel())
    with _on_device(q):
        lib.cbnb_b200_int8_zero_columns(q.data_ptr(), cols.data_ptr(), int(cols.numel()), rows, q.shape[-1], _stream(q))
    lib.check("int8_zero_columns")


def int8_dequant_rows(CB: torch.Tensor, SCB: torch.Tensor, dtype: torch.dtype,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The weight of LLM.int8()'s input gradient, ``W[n, k] = dtype(CB[n, k] * (SCB[n] * (1/127)))``, in one pass: the
    bits of ``CB.to(dtype, copy=True).mul_(SCB.unsqueeze(1).mul(1.0 / 127.0))`` for fp16 / bf16.  ``CB`` is int8
    ``[rows, cols]``, ``SCB`` fp32 ``[rows]``; ``out`` may be a ``[rows, cols]`` view with unit column stride and any row
    stride."""
    if CB.dtype != torch.int8 or CB.dim() != 2:
        raise RuntimeError(f"int8_dequant_rows: CB must be a 2-D int8 tensor, got {CB.dtype} {tuple(CB.shape)}")
    rows, cols = CB.shape
    if SCB.dtype != torch.float32 or SCB.shape != (rows,) or SCB.device != CB.device:
        raise RuntimeError(f"int8_dequant_rows: SCB must be float32 [{rows}] on {CB.device}, got {SCB.dtype} "
                           f"{tuple(SCB.shape)} on {SCB.device}")
    if dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError(f"int8_dequant_rows: dtype must be float16 or bfloat16, got {dtype}")
    if out is None:
        out = torch.empty((rows, cols), device=CB.device, dtype=dtype)
    elif (out.dtype != dtype or out.shape != (rows, cols) or out.device != CB.device
          or (rows > 1 and out.stride(0) < cols) or (cols > 1 and out.stride(1) != 1)):
        raise RuntimeError(f"int8_dequant_rows: out must be {dtype} [{rows}, {cols}] with unit column stride and row "
                           f"stride >= {cols} on {CB.device}")
    ldo = out.stride(0) if rows > 1 else cols
    _check_sizes("int8_dequant_rows", rows, cols, ldo)
    if rows == 0 or cols == 0:
        return out
    CB, SCB = CB.contiguous(), SCB.contiguous()
    with _on_device(CB):
        rc = lib.cbnb_b200_int8_dequant_rows(CB.data_ptr(), SCB.data_ptr(), out.data_ptr(), ldo, rows, cols,
                                             _DTYPE_ID[dtype], _stream(CB))
    lib.check("int8_dequant_rows")
    if rc != 0:
        raise RuntimeError(f"int8_dequant_rows: the library refused the call (code {rc})")
    return out


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
            int8_zero_columns(q, outlier_cols)
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


# outlier columns the operands of the capturable route hold; the GEMM gathers any further ones from A and CB
INT8_OUTLIER_CAPACITY = 64


def int8_outlier_compact(col_flags: torch.Tensor):
    """(cols, count): the flagged columns of ``col_flags`` (int32 [K]) in ascending order in ``cols[:count]`` (int32
    [K]), and their number in ``count`` (int32 [1]), both on the device and without a host synchronisation."""
    if col_flags.dtype != torch.int32 or col_flags.ndim != 1 or not col_flags.is_contiguous():
        raise ValueError("col_flags must be a contiguous 1-D int32 tensor")
    K = col_flags.numel()
    _check_sizes("int8_outlier_compact", K)
    cols = torch.empty(K, device=col_flags.device, dtype=torch.int32)
    count = torch.empty(1, device=col_flags.device, dtype=torch.int32)
    with _on_device(col_flags):
        lib.cbnb_b200_int8_outlier_compact(col_flags.data_ptr(), K, cols.data_ptr(), count.data_ptr(), _stream(col_flags))
    lib.check("int8_outlier_compact")
    return cols, count


def int8_mixed_mm_flags(A, CA, CB, SCA, SCB, col_flags, bias=None) -> torch.Tensor:
    """LLM.int8() forward from the outlier *flags*, with no host synchronisation and no allocation whose size depends
    on the data, so that it can be captured in a CUDA graph and replayed for any outlier set.

    A: fp16 / bf16 activations [..., K]; CA / SCA: their row codes and statistics with ``col_flags`` (int32 [K]) from
    :func:`int8_vectorwise_quant_flags`; CB / SCB: the weight codes [N, K] and statistics.  CA (contiguous) is zeroed
    in place in the outlier columns, as the eager route does.  Returns ``out`` [..., N] of A's dtype: for up to 64
    outlier columns bit-identical to ``int8_mixed_scaled_mm``, beyond that the same formula summed in column order.
    The outlier column indices are not returned."""
    dtype = A.dtype
    if dtype not in (torch.float16, torch.bfloat16):
        raise ValueError(f"int8_mixed_mm_flags: A must be float16 or bfloat16, got {dtype}")
    if CA.dtype != torch.int8 or CB.dtype != torch.int8 or CB.ndim != 2:
        raise ValueError("int8_mixed_mm_flags: CA and CB must be int8, CB of shape [N, K]")
    if SCA.dtype != torch.float32 or SCB.dtype != torch.float32:
        raise ValueError("int8_mixed_mm_flags: SCA and SCB must be float32")
    if bias is not None and (bias.dtype != dtype or bias.ndim != 1):
        raise ValueError(f"int8_mixed_mm_flags: bias must be 1-D of A's dtype {dtype}, got {bias.dtype}")
    N, K = CB.shape
    if K % 16 != 0:
        raise ValueError(f"int8_mixed_mm_flags: K = {K} is not a multiple of 16")
    if A.shape[-1] != K or CA.shape != A.shape or not CA.is_contiguous():
        raise ValueError(f"int8_mixed_mm_flags: A {tuple(A.shape)} and contiguous CA {tuple(CA.shape)} must be [..., {K}]")
    if col_flags.shape != (K,):
        raise ValueError(f"int8_mixed_mm_flags: col_flags must have shape ({K},), got {tuple(col_flags.shape)}")
    M = CA.numel() // K
    _check_sizes("int8_mixed_mm_flags", M, N, K)
    out = torch.empty((*A.shape[:-1], N), device=A.device, dtype=dtype)
    if M == 0:
        return out
    A2 = A.reshape(M, K).contiguous()
    CB = CB.contiguous()
    SCA = SCA.contiguous()
    SCB = SCB.contiguous()
    bias = bias.contiguous() if bias is not None else None
    cols, count = int8_outlier_compact(col_flags)
    subA = torch.empty((M, INT8_OUTLIER_CAPACITY), device=A.device, dtype=dtype)
    subBT = torch.empty((N, INT8_OUTLIER_CAPACITY), device=A.device, dtype=dtype)
    with _on_device(A):
        lib.cbnb_b200_int8_outlier_prep_dev(A2.data_ptr(), CA.data_ptr(), CB.data_ptr(), SCB.data_ptr(), cols.data_ptr(),
                                            count.data_ptr(), M, N, K, _DTYPE_ID[dtype], subA.data_ptr(),
                                            subBT.data_ptr(), _stream(A))
        rc = lib.cbnb_b200_int8_mixed_mm_dev(CA.data_ptr(), CB.data_ptr(), SCA.data_ptr(), SCB.data_ptr(),
                                             bias.data_ptr() if bias is not None else None, A2.data_ptr(),
                                             subA.data_ptr(), subBT.data_ptr(), cols.data_ptr(), count.data_ptr(),
                                             out.data_ptr(), M, N, K, _DTYPE_ID[dtype], _stream(A))
    lib.check("int8_mixed_mm_flags")
    if rc != 0:
        raise RuntimeError(f"int8_mixed_mm_flags: the int8 GEMM does not take this shape (code {rc}): "
                           f"A={tuple(A.shape)} CB={tuple(CB.shape)}")
    return out


@kernel("int8_grouped_mm")
def _int8_grouped_mm(A, CB, SCB, offs, threshold=0.0, bias=None):
    return int8_grouped_mm(A, CB, SCB, offs, threshold, bias)


def int8_grouped_mm(A, CB, SCB, offs, threshold=0.0, bias=None) -> torch.Tensor:
    """LLM.int8() over every expert of a mixture-of-experts layer in one GEMM launch.  ``A [M, K]`` holds the
    expert-sorted rows, ``CB [E, N, K]`` / ``SCB [E * N]`` the expert tensor quantised row-wise as one tensor, ``offs``
    the int32 ``[E]`` end rows (clamped on the device), ``bias`` an optional ``[E, N]``.  The rows of expert e are bit
    for bit what the inference ``Linear8bitLt`` (same threshold) computes on them alone, with each expert's own outlier
    columns; rows past ``offs[E-1]`` are +0.  Nothing is read back to the host and no allocation depends on the data,
    so the call can be captured in a CUDA graph and replayed for any routing and any outlier sets."""
    E, N, K = check_int8_grouped(A, CB, SCB, offs, threshold, bias)
    M = A.shape[0]
    _check_sizes("int8_grouped_mm", M, E * N, K, M * K, E * K, E * N * INT8_OUTLIER_CAPACITY)
    out = torch.empty((M, N), dtype=A.dtype, device=A.device)
    if M == 0:
        return out
    A, CB, SCB, offs = A.contiguous(), CB.contiguous(), SCB.contiguous(), offs.contiguous()
    bias = bias.contiguous() if bias is not None else None
    dtype, stream, dev = _DTYPE_ID[A.dtype], _stream(A), A.device
    # the row codes and statistics of A as fp16, as MatMul8bitLt quantises it (outlier entries -> 0 codes)
    A16 = A if A.dtype == torch.float16 else A.to(torch.float16)
    CA = torch.empty((M, K), device=dev, dtype=torch.int8)
    SCA = torch.empty(M, device=dev, dtype=torch.float32)
    outl = [None] * 5  # A, subA, subBT, cols, count
    with _on_device(A):
        lib.cbnb_b200_int8_vector_quant_flags(A16.data_ptr(), CA.data_ptr(), SCA.data_ptr(), None, float(threshold), M,
                                              K, _DTYPE_ID[torch.float16], stream)
        lib.check("int8_grouped_mm")
        if threshold > 0.0:
            ends = torch.empty(E, device=dev, dtype=torch.int32)
            flags = torch.empty((E, K), device=dev, dtype=torch.int32)
            cols = torch.empty((E, K), device=dev, dtype=torch.int32)
            count = torch.empty(E, device=dev, dtype=torch.int32)
            subA = torch.empty((M, INT8_OUTLIER_CAPACITY), device=dev, dtype=A.dtype)
            subBT = torch.empty((E * N, INT8_OUTLIER_CAPACITY), device=dev, dtype=A.dtype)
            rc = lib.cbnb_b200_int8_grouped_outliers(A.data_ptr(), A16.data_ptr(), CA.data_ptr(), CB.data_ptr(),
                                                     SCB.data_ptr(), offs.data_ptr(), E, float(threshold),
                                                     ends.data_ptr(), flags.data_ptr(), cols.data_ptr(),
                                                     count.data_ptr(), subA.data_ptr(), subBT.data_ptr(), M, N, K,
                                                     dtype, stream)
            lib.check("int8_grouped_mm")
            if rc != 0:
                raise RuntimeError(f"int8_grouped_mm: the library refused the outlier preparation (code {rc})")
            outl = [t.data_ptr() for t in (A, subA, subBT, cols, count)]
        rc = lib.cbnb_b200_int8_grouped_mm(CA.data_ptr(), CB.data_ptr(), SCA.data_ptr(), SCB.data_ptr(),
                                           bias.data_ptr() if bias is not None else None, offs.data_ptr(), E, *outl,
                                           out.data_ptr(), M, N, K, dtype, stream)
    lib.check("int8_grouped_mm")
    if rc != 0:
        raise RuntimeError(f"int8_grouped_mm: the library does not serve this call (code {rc}): A={tuple(A.shape)} "
                           f"CB={tuple(CB.shape)}")
    return out


# ------------------------------------------------------------------------------------------ tensor-parallel LLM.int8()
def _int8_acts(what: str, A: torch.Tensor) -> tuple[torch.Tensor, int, int]:
    if A.dtype not in (torch.float16, torch.bfloat16) or not A.is_cuda:
        raise ValueError(f"{what}: A must be a float16 or bfloat16 CUDA tensor, got {A.dtype} on {A.device}")
    cols = A.shape[-1]
    rows = A.numel() // cols if cols else 0
    _check_sizes(what, rows, cols)
    return A.contiguous(), rows, cols


def int8_row_stats(A: torch.Tensor, threshold: float):
    """(row_stats fp32 [rows], col_flags int32 [cols] or None): the statistics half of
    :func:`int8_vectorwise_quant_flags` -- the absmax of each row over the entries below ``threshold`` and the columns
    holding an entry at or above it -- without the codes."""
    A, rows, cols = _int8_acts("int8_row_stats", A)
    if threshold < 0.0:
        raise ValueError("int8_row_stats: threshold must be non-negative")
    row_stats = torch.empty(rows, device=A.device, dtype=torch.float32)
    flags = torch.zeros(cols, device=A.device, dtype=torch.int32) if threshold > 0.0 else None
    if rows == 0:
        return row_stats, flags
    with _on_device(A):
        rc = lib.cbnb_b200_int8_row_stats(A.data_ptr(), row_stats.data_ptr(),
                                          flags.data_ptr() if flags is not None else None, float(threshold), rows, cols,
                                          _DTYPE_ID[A.dtype], _stream(A))
    lib.check("int8_row_stats")
    if rc != 0:
        raise RuntimeError(f"int8_row_stats: the library refused the call (code {rc})")
    return row_stats, flags


def int8_quant_with_stats(A: torch.Tensor, row_stats: torch.Tensor, threshold: float) -> torch.Tensor:
    """The codes half of :func:`int8_vectorwise_quant_flags`: ``int8(rint(A * (127 / row_stats)))`` with the kernel's
    rounding, entries at or above ``threshold`` -> 0, for given statistics (fp32 [rows] on A's device)."""
    A, rows, cols = _int8_acts("int8_quant_with_stats", A)
    if row_stats.dtype != torch.float32 or row_stats.shape != (rows,) or row_stats.device != A.device:
        raise ValueError(f"int8_quant_with_stats: row_stats must be float32 [{rows}] on {A.device}")
    q = torch.empty(A.shape, device=A.device, dtype=torch.int8)
    if rows == 0:
        return q
    row_stats = row_stats.contiguous()
    with _on_device(A):
        rc = lib.cbnb_b200_int8_quant_with_stats(A.data_ptr(), q.data_ptr(), row_stats.data_ptr(), float(threshold),
                                                 rows, cols, _DTYPE_ID[A.dtype], _stream(A))
    lib.check("int8_quant_with_stats")
    if rc != 0:
        raise RuntimeError(f"int8_quant_with_stats: the library refused the call (code {rc})")
    return q


def _dest_ptrs(what: str, outs, dtype: torch.dtype, device, M: int, N: int, ldc: int, exc=ValueError) -> list[int]:
    """Device addresses of 1..8 destinations of an [M, N] output at row stride ``ldc``: tensors (checked: dtype,
    device, room for the output) or raw addresses of peers' symmetric-memory buffers, which the caller vouches for.
    Raises ``exc`` (each public wrapper keeps its own exception type)."""
    if not 1 <= len(outs) <= 8:
        raise exc(f"{what}: between 1 and 8 destinations, got {len(outs)}")
    if ldc < N:
        raise exc(f"{what}: ldc ({ldc}) < N ({N})")
    need = (M - 1) * ldc + N if M > 0 else 0
    ptrs = []
    for o in outs:
        if isinstance(o, torch.Tensor):
            if o.dtype != dtype or o.device != device:
                raise exc(f"{what}: destinations must be {dtype} on {device}, got {o.dtype} on {o.device}")
            if o.untyped_storage().nbytes() // o.element_size() - o.storage_offset() < need:
                raise exc(f"{what}: a destination needs {need} elements from its start")
            ptrs.append(o.data_ptr())
        else:
            ptrs.append(int(o))
    return ptrs


def _outlier_operands(what: str, subA, subBT, M: int, N: int, dtype) -> int:
    """jpad of the padded outlier operands subA [M, jpad] / subBT [N, jpad] (0 when both are None)."""
    if subA is None and subBT is None:
        return 0
    if subA is None or subBT is None:
        raise ValueError(f"{what}: subA and subBT go together")
    jpad = subA.shape[-1] if subA.dim() == 2 else -1
    if (subA.dtype != dtype or subBT.dtype != dtype or subA.shape != (M, jpad) or subBT.shape != (N, jpad)
            or not subA.is_contiguous() or not subBT.is_contiguous()):
        raise ValueError(f"{what}: subA / subBT must be contiguous {dtype} [{M}, jpad] / [{N}, jpad]")
    if not 8 <= jpad <= 64 or jpad % 8 != 0:
        raise ValueError(f"{what}: jpad must be a multiple of 8 in [8, 64], got {jpad}")
    if subA.data_ptr() % 16 or subBT.data_ptr() % 16:
        raise ValueError(f"{what}: subA / subBT must be 16-byte aligned")
    return jpad


def int8_gemm_multi_out(CA, CB, SCA, SCB, outs, ldc: int, dtype: Optional[torch.dtype], bias=None, subA=None,
                        subBT=None) -> bool:
    """The int8 GEMM storing every output element to each destination in ``outs`` (row stride ``ldc``): dtype None
    gives the int32 accumulators (``int8_linear_matmul``), float16 / bfloat16 the fused epilogue of ``int8_scaled_mm``,
    plus with ``subA`` [M, jpad] / ``subBT`` [N, jpad] (from :func:`int8_outlier_operands`, zero-padded) the outlier term
    of ``int8_mixed_scaled_mm``.  Each destination holds the single-destination bits.  Returns False when the kernel
    does not take the shape (K % 16, alignment): the caller takes another route."""
    if CA.dtype != torch.int8 or CB.dtype != torch.int8 or CB.dim() != 2:
        raise ValueError("int8_gemm_multi_out: CA and CB must be int8, CB of shape [N, K]")
    N, K = CB.shape
    if CA.shape[-1] != K:
        raise ValueError(f"int8_gemm_multi_out: CA {tuple(CA.shape)} does not match CB {tuple(CB.shape)}")
    M = CA.numel() // K if K else 0
    _check_sizes("int8_gemm_multi_out", M, N, K, ldc)
    if dtype is None:
        if bias is not None or subA is not None or subBT is not None:
            raise ValueError("int8_gemm_multi_out: the int32 form takes no bias and no outlier operands")
        epi, out_dtype = 0, torch.int32
    elif dtype in (torch.float16, torch.bfloat16):
        epi, out_dtype = _DTYPE_ID[dtype], dtype
        if SCA.dtype != torch.float32 or SCB.dtype != torch.float32 or SCA.shape != (M,) or SCB.shape != (N,):
            raise ValueError(f"int8_gemm_multi_out: SCA / SCB must be float32 [{M}] / [{N}]")
        if bias is not None and (bias.dtype != dtype or bias.shape != (N,)):
            raise ValueError(f"int8_gemm_multi_out: bias must be {dtype} [{N}]")
    else:
        raise ValueError(f"int8_gemm_multi_out: dtype must be None, float16 or bfloat16, got {dtype}")
    jpad = _outlier_operands("int8_gemm_multi_out", subA, subBT, M, N, dtype)
    ptrs = _dest_ptrs("int8_gemm_multi_out", outs, out_dtype, CA.device, M, N, ldc)
    if M == 0 or N == 0:
        return True
    CA, CB = CA.contiguous(), CB.contiguous()
    SCA = SCA.contiguous() if SCA is not None else None
    SCB = SCB.contiguous() if SCB is not None else None
    bias = bias.contiguous() if bias is not None else None
    arr = (ct.c_void_p * len(ptrs))(*ptrs)
    with _on_device(CA):
        rc = lib.cbnb_b200_int8_gemm_multi_out(
            CA.data_ptr(), CB.data_ptr(), SCA.data_ptr() if SCA is not None else None,
            SCB.data_ptr() if SCB is not None else None, bias.data_ptr() if bias is not None else None,
            subA.data_ptr() if subA is not None else None, subBT.data_ptr() if subBT is not None else None, jpad,
            ct.cast(arr, ct.c_void_p), len(ptrs), M, N, K, ldc, epi, _stream(CA))
    lib.check("int8_gemm_multi_out")
    return rc == 0


def int8_gemm_partial_scatter(CA, CB, outs, ldc: int) -> bool:
    """The exact int32 partial ``CA . CB^T`` with its rows scattered over ``outs`` in rank order: with ``w = len(outs)``
    and ``M`` rows, row ``m`` is stored to ``outs[m // (M/w)]`` at row ``m % (M/w)`` (row stride ``ldc``), the partial of
    a sequence-parallel K-sharded layer whose rank s owns tokens ``[s*M/w, (s+1)*M/w)``.  Same kernel and bits as
    :func:`int8_gemm_multi_out` with dtype None.  ``M % w == 0`` is required.  A destination is an int32 CUDA tensor,
    checked here, or a raw device address, which the caller vouches for.  Returns False when the kernel does not take
    the shape (K % 16, alignment)."""
    if CA.dtype != torch.int8 or CB.dtype != torch.int8 or CB.dim() != 2:
        raise RuntimeError("int8_gemm_partial_scatter: CA and CB must be int8, CB of shape [N, K]")
    N, K = CB.shape
    if CA.shape[-1] != K:
        raise RuntimeError(f"int8_gemm_partial_scatter: CA {tuple(CA.shape)} does not match CB {tuple(CB.shape)}")
    M = CA.numel() // K if K else 0
    _check_sizes("int8_gemm_partial_scatter", M, N, K, ldc)
    n = len(outs)
    if n < 1 or M < n or M % n != 0:
        raise RuntimeError(f"int8_gemm_partial_scatter: {M} rows do not split evenly over {n} destinations")
    ptrs = _dest_ptrs("int8_gemm_partial_scatter", outs, torch.int32, CA.device, M // n, N, ldc, RuntimeError)
    if N == 0:
        return True
    CA, CB = CA.contiguous(), CB.contiguous()
    arr = (ct.c_void_p * n)(*ptrs)
    with _on_device(CA):
        rc = lib.cbnb_b200_int8_gemm_partial_scatter(CA.data_ptr(), CB.data_ptr(), ct.cast(arr, ct.c_void_p), n, M // n,
                                                     M, N, K, ldc, _stream(CA))
    lib.check("int8_gemm_partial_scatter")
    return rc == 0


def int8_outlier_operands(A, CB, SCB, cols: torch.Tensor, jpad: Optional[int] = None):
    """(subA [M, jpad], subBT [N, jpad]) of A's dtype: ``subA[m, j] = A[m, cols[j]]`` and ``subBT[n, j] = T((CB[n,
    cols[j]] * SCB[n]) * (1/127))``, as the fused LLM.int8() route builds them, zero past ``len(cols)``.  ``jpad``
    defaults to ``len(cols)`` rounded up to a multiple of 8."""
    dtype = A.dtype
    if dtype not in (torch.float16, torch.bfloat16):
        raise ValueError(f"int8_outlier_operands: A must be float16 or bfloat16, got {dtype}")
    if CB.dtype != torch.int8 or CB.dim() != 2 or SCB.dtype != torch.float32 or SCB.shape != (CB.shape[0],):
        raise ValueError("int8_outlier_operands: CB must be int8 [N, K] and SCB float32 [N]")
    N, K = CB.shape
    if A.shape[-1] != K:
        raise ValueError(f"int8_outlier_operands: A {tuple(A.shape)} does not match CB {tuple(CB.shape)}")
    J = int(cols.numel())
    jpad = -(-J // 8) * 8 if jpad is None else jpad
    if jpad < J or jpad % 8 != 0:
        raise ValueError(f"int8_outlier_operands: jpad ({jpad}) must be a multiple of 8 >= {J}")
    M = A.numel() // K if K else 0
    _check_sizes("int8_outlier_operands", M, N, K, jpad)
    subA = torch.zeros((M, jpad), device=A.device, dtype=dtype)
    subBT = torch.zeros((N, jpad), device=A.device, dtype=dtype)
    if jpad == 0 or M + N == 0:
        return subA, subBT
    A2 = A.reshape(M, K).contiguous()
    cols = cols.to(device=A.device, dtype=torch.int64).contiguous()
    with _on_device(A):
        lib.cbnb_b200_int8_outlier_prep(A2.data_ptr(), CB.contiguous().data_ptr(), SCB.contiguous().data_ptr(),
                                        cols.data_ptr(), J, jpad, M, N, K, _DTYPE_ID[dtype], subA.data_ptr(),
                                        subBT.data_ptr(), _stream(A))
    lib.check("int8_outlier_operands")
    return subA, subBT


def int8_reduce_partials(parts: torch.Tensor, SCA, SCB, dtype: torch.dtype, bias=None, subA=None, subBT=None,
                         out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out = epilogue(parts[0] + ... + parts[w-1])``: the exact int32 partials ``[w, M, N]`` of a K-sharded LLM.int8()
    layer summed, then dequantised exactly as the int8 GEMM's epilogue does (``SCA`` [M], ``SCB`` [N], the bias rules of
    fp16 / bf16 output), with the outlier term of ``subA`` [M, jpad] / ``subBT`` [N, jpad] when given.  ``out`` may be
    an ``[M, N]`` view with unit column stride and any row stride."""
    if parts.dtype != torch.int32 or parts.dim() != 3 or not parts.is_cuda:
        raise ValueError(f"int8_reduce_partials: parts must be a [world, M, N] int32 CUDA tensor, got {parts.dtype} "
                         f"{tuple(parts.shape)} on {parts.device}")
    if dtype not in (torch.float16, torch.bfloat16):
        raise ValueError(f"int8_reduce_partials: dtype must be float16 or bfloat16, got {dtype}")
    world, M, N = parts.shape
    if world < 1:
        raise ValueError("int8_reduce_partials: no partials")
    if (SCA.dtype != torch.float32 or SCB.dtype != torch.float32 or SCA.shape != (M,) or SCB.shape != (N,)
            or SCA.device != parts.device or SCB.device != parts.device):
        raise ValueError(f"int8_reduce_partials: SCA / SCB must be float32 [{M}] / [{N}] on {parts.device}")
    if bias is not None and (bias.dtype != dtype or bias.shape != (N,) or bias.device != parts.device):
        raise ValueError(f"int8_reduce_partials: bias must be {dtype} [{N}] on {parts.device}")
    jpad = _outlier_operands("int8_reduce_partials", subA, subBT, M, N, dtype)
    if out is None:
        out = torch.empty((M, N), dtype=dtype, device=parts.device)
    elif (out.dtype != dtype or out.shape != (M, N) or out.device != parts.device
          or (M > 1 and out.stride(1) != 1) or out.stride(0) < N):
        raise ValueError(f"int8_reduce_partials: out must be {dtype} [{M}, {N}] with unit column stride on "
                         f"{parts.device}")
    _check_sizes("int8_reduce_partials", M, N, out.stride(0), world)
    if M == 0 or N == 0:
        return out
    parts = parts.contiguous()
    SCA, SCB = SCA.contiguous(), SCB.contiguous()
    bias = bias.contiguous() if bias is not None else None
    with _on_device(parts):
        rc = lib.cbnb_b200_int8_reduce_partials(
            parts.data_ptr(), world, M * N, SCA.data_ptr(), SCB.data_ptr(), bias.data_ptr() if bias is not None else None,
            subA.data_ptr() if subA is not None else None, subBT.data_ptr() if subBT is not None else None, jpad,
            out.data_ptr(), M, N, out.stride(0), _DTYPE_ID[dtype], _stream(parts))
    lib.check("int8_reduce_partials")
    if rc != 0:
        raise RuntimeError(f"int8_reduce_partials: the library refused the call (code {rc})")
    return out


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


# ---- multi-tensor steps: one native call per descriptor-capacity chunk of a list of tensors that share every scalar
_multi_capacity = None


def optimizer_multi_capacity() -> int:
    """Tensors per multi-tensor launch: the descriptors travel as a kernel parameter (at most 32764 bytes)."""
    global _multi_capacity
    if _multi_capacity is None:
        _multi_capacity = int(lib.cbnb_b200_optimizer_multi_capacity())
    return _multi_capacity


def _optimizer_list(what, optimizer_name, supported, g, p, state1, state2, absmax1, absmax2, step, eight_bit):
    """Validate a multi-tensor step as the single-tensor ops do and pack its descriptors (cextension.OptimTensor).
    Returns (g[0], descriptors, capturable): capturable when the steps are CUDA tensors, the device step counters that
    the _dev entries advance and read; their descriptors carry the counters' pointers instead of the steps."""
    if optimizer_name not in supported:
        raise ValueError(f"Unsupported optimizer name: {optimizer_name}. Supported optimizers: {list(supported)}")
    k = len(p)
    two = optimizer_name in ("adam", "ademamix", "lamb")
    lists = {"g": g, "state1": state1, "step": step}
    if two:
        lists["state2"] = state2
    if eight_bit:
        lists["absmax1"] = absmax1
        if two:
            lists["absmax2"] = absmax2
    for name, values in lists.items():
        if values is None or len(values) != k:
            raise ValueError(f"{what}: {name} must list one entry per parameter ({k})")
    if k == 0:
        return None, None, False
    dtype, device = g[0].dtype, g[0].device
    capturable = any(isinstance(s, torch.Tensor) and s.is_cuda for s in step)
    if dtype not in _DTYPE_ID:
        raise ValueError(f"{what}: unsupported gradient dtype {dtype}. Supported dtypes: torch.float32, torch.float16, "
                         "torch.bfloat16")
    if device.type != "cuda":
        raise RuntimeError(f"{what}: tensors must live on a CUDA device, got {device}")
    descs, step_ptrs = [], set()
    for i in range(k):
        s2 = state2[i] if two else None
        a1 = absmax1[i] if eight_bit else None
        a2 = absmax2[i] if eight_bit and two else None
        gi, pi = g[i], p[i]
        if gi.dtype != dtype or pi.dtype != dtype or gi.numel() != pi.numel():
            raise ValueError(f"{what}: every g and p must have dtype {dtype} and g and p the same number of elements "
                             f"(entry {i}: {gi.dtype} {tuple(gi.shape)}, {pi.dtype} {tuple(pi.shape)})")
        for t in (gi, pi, state1[i], s2, a1, a2):
            if t is None:
                continue
            if not t.is_contiguous():
                raise ValueError(f"{what}: tensors must be contiguous (entry {i})")
            # managed ("paged") state is a CPU tensor to PyTorch that every GPU can address
            if t.device != device and not getattr(t, "is_paged", False):
                raise RuntimeError(f"{what}: tensors must be on one device, {device}; entry {i} has one on {t.device}")
        if not capturable:
            descs.append(cext.OptimTensor(pi.data_ptr(), gi.data_ptr(), state1[i].data_ptr(), _optional_ptr(s2),
                                          _optional_ptr(a1), _optional_ptr(a2), pi.numel(), int(step[i]), 0))
            continue
        si = step[i]
        if (not isinstance(si, torch.Tensor) or si.dtype != torch.int32 or si.numel() != 1 or not si.is_contiguous()
                or si.device != device):
            raise ValueError(f"{what}: device steps must be contiguous one-element int32 tensors on {device} (entry {i})")
        d = cext.OptimTensor(pi.data_ptr(), gi.data_ptr(), state1[i].data_ptr(), _optional_ptr(s2), _optional_ptr(a1),
                             _optional_ptr(a2), pi.numel())
        d.step_ptr = si.data_ptr()
        step_ptrs.add(d.step_ptr)
        descs.append(d)
    if capturable and len(step_ptrs) != k:
        raise ValueError(f"{what}: every parameter needs its own step counter (the call advances each once)")
    return g[0], (cext.OptimTensor * k)(*descs), capturable


def _device_lr(what, lr, device):
    """(lr, lr_dev) of a capturable call: a one-element fp32 tensor on the device is read by the kernel at every launch
    (and every replay of a CUDA graph); a number is passed by value."""
    if not isinstance(lr, torch.Tensor):
        return float(lr), None
    if lr.dtype != torch.float32 or lr.numel() != 1 or lr.device != device:
        raise ValueError(f"{what}: a tensor lr must be a one-element float32 tensor on {device}, got {lr.dtype} "
                         f"{tuple(lr.shape)} on {lr.device}")
    return 0.0, lr.data_ptr()


def _launch_list(what, fn, optimizer_name, g0, descs, scalars):
    """fn(optimizer, dtype, tensors, count, *scalars, stream) once per capacity chunk of descs."""
    cap, k, size = optimizer_multi_capacity(), len(descs), ct.sizeof(cext.OptimTensor)
    for lo in range(0, k, cap):
        rc = fn(_OPTIMIZER_ID[optimizer_name], _DTYPE_ID[g0.dtype], ct.addressof(descs) + lo * size, min(cap, k - lo),
                *scalars, _stream(g0))
        lib.check(what)
        if rc != 0:
            raise RuntimeError(f"{what}: native call returned {rc}")


def optimizer_update_32bit_multi(optimizer_name, g, p, state1, state2, beta1, beta2, beta3, alpha, eps, weight_decay, step,
                                 lr, gnorm_scale=1.0, skip_zeros=False):
    """In-place fp32-state steps of several parameters in one launch per capacity chunk: g, p, state1, state2 (None for
    one-state optimizers) and step list one entry per parameter; the scalars are shared.  No trust ratio (max_unorm).

    Capturable route: when the steps are one-element int32 CUDA tensors, the call advances each by one on the device
    and updates with the advanced values; lr may then also be a one-element fp32 CUDA tensor.  Nothing is read on the
    host, so the call can be captured in a CUDA graph and replayed."""
    what = "optimizer_update_32bit_multi"
    g0, descs, dev = _optimizer_list(what, optimizer_name, _OPTIMIZER_ID, g, p, state1, state2, None, None, step, False)
    if descs is None:
        return
    if dev:
        lr_value, lr_dev = _device_lr(what, lr, g0.device)
        fn, scalars = lib.cbnb_b200_optimizer_update_32bit_multi_dev, (float(lr_value), lr_dev)
    else:
        fn, scalars = lib.cbnb_b200_optimizer_update_32bit_multi, (float(lr),)
    with _on_device(g0):
        _launch_list(what, fn, optimizer_name, g0, descs,
                     (float(beta1), float(beta2), float(beta3), float(alpha), float(eps), float(weight_decay), *scalars,
                      float(gnorm_scale), bool(skip_zeros)))


def optimizer_update_8bit_blockwise_multi(optimizer_name, g, p, state1, state2, beta1, beta2, beta3, alpha, eps, step, lr,
                                          qmap1, qmap2, absmax1, absmax2, weight_decay, gnorm_scale=1.0, skip_zeros=False):
    """In-place blockwise (256) 8-bit-state steps of several parameters in one launch per capacity chunk: g, p, state1,
    state2, absmax1, absmax2 and step list one entry per parameter (state2 / absmax2 None for one-state optimizers);
    the code books qmap1 / qmap2 and the scalars are shared.  Device steps (and lr) as optimizer_update_32bit_multi."""
    what = "optimizer_update_8bit_blockwise_multi"
    g0, descs, dev = _optimizer_list(what, optimizer_name, _OPTIMIZER_8BIT, g, p, state1, state2, absmax1, absmax2, step,
                                     True)
    if descs is None:
        return
    two = optimizer_name in ("adam", "ademamix")
    for q in (qmap1, qmap2) if two else (qmap1,):
        if q is None or q.device != g0.device or not q.is_contiguous() or q.dtype != torch.float32 or q.numel() < 256:
            raise ValueError(f"{what}: the code books must be contiguous fp32 [256] tensors on {g0.device}")
    if dev:
        lr_value, lr_dev = _device_lr(what, lr, g0.device)
        fn, scalars = lib.cbnb_b200_optimizer_update_8bit_blockwise_multi_dev, (float(lr_value), lr_dev)
    else:
        fn, scalars = lib.cbnb_b200_optimizer_update_8bit_blockwise_multi, (float(lr),)
    with _on_device(g0):
        _launch_list(what, fn, optimizer_name, g0, descs,
                     (float(beta1), float(beta2), float(beta3), float(alpha), float(eps), float(weight_decay), *scalars,
                      qmap1.data_ptr(), qmap2.data_ptr() if two else None, float(gnorm_scale), bool(skip_zeros)))


# ---- data-parallel steps: one rank's pieces of flat gradient / parameter buffers, gradients summed over the ranks
_OPTIMIZER_PEERS = tuple(name for name in _OPTIMIZER_ID if name != "ademamix")
_peers_capacity = None


def optimizer_peers_capacity() -> int:
    """Pieces per data-parallel launch: the descriptor list shares the kernel parameters with the peer addresses."""
    global _peers_capacity
    if _peers_capacity is None:
        _peers_capacity = int(lib.cbnb_b200_optimizer_peers_capacity())
    return _peers_capacity


def _peer_args(what, g, p, step, grad_srcs, param_dsts, grad_local, param_local):
    """Check the peer arguments: 1..8 sources and destinations (addresses) and the local flat buffers holding every
    piece (g[i] inside grad_local, p[i] inside param_local).  Returns the two address arrays.  (step, host steps or
    device counters, is checked by _optimizer_list.)"""
    srcs, dsts = [int(a) for a in grad_srcs], [int(a) for a in param_dsts]
    if not 1 <= len(srcs) <= 8 or not 1 <= len(dsts) <= 8:
        raise ValueError(f"{what}: {len(srcs)} gradient sources and {len(dsts)} parameter destinations (1..8 each)")
    if any(a == 0 for a in srcs + dsts):
        raise ValueError(f"{what}: a null gradient source or parameter destination")
    for name, flat in (("grad_local", grad_local), ("param_local", param_local)):
        if (not isinstance(flat, torch.Tensor) or not flat.is_contiguous() or flat.dtype != grad_local.dtype
                or flat.numel() != grad_local.numel() or flat.device != grad_local.device):
            raise ValueError(f"{what}: {name} must be a contiguous flat buffer like grad_local")
    es = grad_local.element_size()
    for i, (gi, pi) in enumerate(zip(g, p)):
        for t, flat in ((gi, grad_local), (pi, param_local)):
            off = t.data_ptr() - flat.data_ptr()
            if t.dtype != flat.dtype or off < 0 or off % es or off // es + t.numel() > flat.numel():
                raise ValueError(f"{what}: piece {i} is not a {flat.dtype} view inside the local flat buffers")
    return (ct.c_void_p * len(srcs))(*srcs), (ct.c_void_p * len(dsts))(*dsts)


def _launch_peers(what, fn, optimizer_name, g0, descs, srcs, dsts, grad_local, param_local, grad_scale, scalars):
    """fn(optimizer, dtype, tensors, count, srcs, world, dsts, ndst, grad_local, param_local, numel, grad_scale,
    *scalars, stream) once per capacity chunk of descs."""
    cap, k, size = optimizer_peers_capacity(), len(descs), ct.sizeof(cext.OptimTensor)
    for lo in range(0, k, cap):
        rc = fn(_OPTIMIZER_ID[optimizer_name], _DTYPE_ID[g0.dtype], ct.addressof(descs) + lo * size, min(cap, k - lo),
                ct.cast(srcs, ct.c_void_p), len(srcs), ct.cast(dsts, ct.c_void_p), len(dsts), grad_local.data_ptr(),
                param_local.data_ptr(), grad_local.numel(), float(grad_scale), *scalars, _stream(g0))
        lib.check(what)
        if rc != 0:
            raise RuntimeError(f"{what}: native call returned {rc}")


def _gnorm_scale_dev(what, gnorm_scale_dev, device):
    """The address of a device-side gradient factor: a one-element fp32 tensor on the gradients' device."""
    t = gnorm_scale_dev
    if (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.numel() != 1 or t.device != device):
        raise ValueError(f"{what}: gnorm_scale_dev must be a one-element float32 tensor on {device}")
    return t.data_ptr()


def _peers_entry(what, dev, lr, gnorm_scale_dev, device):
    """(name, lr, trailing pointer arguments) of the entry a data-parallel step calls: ``what``_dev for device steps
    (dev: lr may be a tensor, lr_dev; the coefficient may be NULL), ``what``_scaled with a coefficient, else ``what``."""
    if dev:
        what += "_dev"
        lr, lr_dev = _device_lr(what, lr, device)
        coef = None if gnorm_scale_dev is None else _gnorm_scale_dev(what, gnorm_scale_dev, device)
        return what, lr, (coef, lr_dev)
    if gnorm_scale_dev is None:
        return what, float(lr), ()
    what += "_scaled"
    return what, float(lr), (_gnorm_scale_dev(what, gnorm_scale_dev, device),)


def optimizer_update_32bit_multi_peers(optimizer_name, g, p, state1, state2, beta1, beta2, beta3, alpha, eps,
                                       weight_decay, step, lr, grad_srcs, param_dsts, grad_local, param_local,
                                       grad_scale, skip_zeros=False, gnorm_scale_dev=None):
    """optimizer_update_32bit_multi for one data-parallel rank: g and p list pieces of the local flat buffers grad_local
    and param_local; the gradient of each element is the fp32 sum, in rank order, of the buffers at the addresses
    grad_srcs (each laid out as grad_local) times grad_scale, rounded once to the dtype; the new parameters go to each
    address of param_dsts (laid out as param_local), not to p unless param_local is among them.

    gnorm_scale_dev: a one-element fp32 CUDA tensor (a clip coefficient) that the kernel reads and applies as the
    multi-tensor step applies gnorm_scale; None: 1, no read.

    Capturable route: when the steps are one-element int32 CUDA tensors (each its own), the kernels read them on the
    device and lr may be a one-element fp32 CUDA tensor, as in optimizer_update_32bit_multi; but this call does not
    advance the steps: the caller advances them, on every rank, before the call.  Nothing is read on the host."""
    what = "optimizer_update_32bit_multi_peers"
    g0, descs, dev = _optimizer_list(what, optimizer_name, _OPTIMIZER_PEERS, g, p, state1, state2, None, None, step,
                                     False)
    if descs is None:
        return
    srcs, dsts = _peer_args(what, g, p, step, grad_srcs, param_dsts, grad_local, param_local)
    what, lr, tail = _peers_entry(what, dev, lr, gnorm_scale_dev, g0.device)
    scalars = (float(beta1), float(beta2), float(beta3), float(alpha), float(eps), float(weight_decay), lr,
               bool(skip_zeros)) + tail
    with _on_device(g0):
        _launch_peers(what, getattr(lib, "cbnb_b200_" + what), optimizer_name, g0, descs, srcs, dsts, grad_local,
                      param_local, grad_scale, scalars)


def optimizer_update_8bit_blockwise_multi_peers(optimizer_name, g, p, state1, state2, beta1, beta2, beta3, alpha, eps,
                                                step, lr, qmap1, qmap2, absmax1, absmax2, weight_decay, grad_srcs,
                                                param_dsts, grad_local, param_local, grad_scale, skip_zeros=False,
                                                gnorm_scale_dev=None):
    """optimizer_update_8bit_blockwise_multi for one data-parallel rank; the gradient and parameter exchange, and
    gnorm_scale_dev and device steps (and lr), as optimizer_update_32bit_multi_peers.  Every piece starts on a
    256-element block of its tensor."""
    what = "optimizer_update_8bit_blockwise_multi_peers"
    g0, descs, dev = _optimizer_list(what, optimizer_name, [n for n in _OPTIMIZER_8BIT if n in _OPTIMIZER_PEERS], g, p,
                                   state1, state2, absmax1, absmax2, step, True)
    if descs is None:
        return
    srcs, dsts = _peer_args(what, g, p, step, grad_srcs, param_dsts, grad_local, param_local)
    two = optimizer_name == "adam"
    for q in (qmap1, qmap2) if two else (qmap1,):
        if q is None or q.device != g0.device or not q.is_contiguous() or q.dtype != torch.float32 or q.numel() < 256:
            raise ValueError(f"{what}: the code books must be contiguous fp32 [256] tensors on {g0.device}")
    what, lr, tail = _peers_entry(what, dev, lr, gnorm_scale_dev, g0.device)
    scalars = (float(beta1), float(beta2), float(beta3), float(alpha), float(eps), float(weight_decay), lr,
               qmap1.data_ptr(), qmap2.data_ptr() if two else None, bool(skip_zeros)) + tail
    with _on_device(g0):
        _launch_peers(what, getattr(lib, "cbnb_b200_" + what), optimizer_name, g0, descs, srcs, dsts, grad_local,
                      param_local, grad_scale, scalars)


def optimizer_grad_norm_peers(g, grad_srcs, grad_local, grad_scale, norm_type, acc):
    """Add the norm value of one data-parallel rank's pieces of the reduced gradient into acc (a one-element float64
    CUDA tensor), on the device: the sum of squares (norm_type 2) or the max |g| (norm_type inf) of every element's
    gradient T(fp32 rank-order sum over grad_srcs * grad_scale), formed as the peer steps form it.  g lists pieces of
    the flat buffer grad_local; grad_srcs, as for optimizer_update_32bit_multi_peers.  One launch per capacity chunk,
    each folding into acc in stream order; nothing is read on the host."""
    what = "optimizer_grad_norm_peers"
    inf = _norm_kind(what, norm_type)
    if not isinstance(acc, torch.Tensor) or acc.dtype != torch.float64 or acc.numel() != 1 or not acc.is_cuda:
        raise ValueError(f"{what}: acc must be a one-element float64 CUDA tensor")
    if not g:
        return
    if grad_local.dtype not in _DTYPE_ID or not grad_local.is_cuda or acc.device != grad_local.device:
        raise ValueError(f"{what}: grad_local must be an fp32 / fp16 / bf16 CUDA tensor on acc's device")
    srcs, _ = _peer_args(what, g, g, [], grad_srcs, [grad_local.data_ptr()], grad_local, grad_local)
    descs = (cext.OptimTensor * len(g))(*[cext.OptimTensor(0, t.data_ptr(), 0, 0, 0, 0, t.numel(), 0, 0) for t in g])
    cap, size = optimizer_peers_capacity(), ct.sizeof(cext.OptimTensor)
    with _on_device(grad_local):
        for lo in range(0, len(g), cap):
            rc = lib.cbnb_b200_optimizer_grad_norm_peers(
                _DTYPE_ID[grad_local.dtype], ct.addressof(descs) + lo * size, min(cap, len(g) - lo),
                ct.cast(srcs, ct.c_void_p), len(srcs), grad_local.data_ptr(), grad_local.numel(), float(grad_scale),
                inf, acc.data_ptr(), _stream(grad_local))
            lib.check(what)
            if rc != 0:
                raise RuntimeError(f"{what}: native call returned {rc}")


def optimizer_clip_coef(rank_values, norm_type, max_norm, out):
    """The global gradient norm and clip coefficient from the ranks' values of optimizer_grad_norm_peers (a float64
    CUDA tensor, rank order), on the device: out (two float32 elements) receives the total norm and the coefficient,
    the bits of torch's ``(max_norm / (total_norm + 1e-6)).clamp(max=1.0)`` on that fp32 norm."""
    what = "optimizer_clip_coef"
    inf = _norm_kind(what, norm_type)
    if (not isinstance(rank_values, torch.Tensor) or rank_values.dtype != torch.float64 or not rank_values.is_cuda
            or not rank_values.is_contiguous() or rank_values.numel() < 1):
        raise ValueError(f"{what}: rank_values must be a contiguous float64 CUDA tensor")
    if (not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.numel() != 2 or not out.is_contiguous()
            or out.device != rank_values.device):
        raise ValueError(f"{what}: out must be a contiguous two-element float32 tensor on {rank_values.device}")
    with _on_device(out):
        rc = lib.cbnb_b200_optimizer_clip_coef(rank_values.data_ptr(), rank_values.numel(), inf, float(max_norm),
                                               out.data_ptr(), _stream(out))
    lib.check(what)
    if rc != 0:
        raise RuntimeError(f"{what}: native call returned {rc}")


def _norm_kind(what, norm_type) -> bool:
    """True for the inf norm, False for L2; any other order is refused."""
    t = float(norm_type)
    if t not in (2.0, float("inf")):
        raise ValueError(f"{what}: norm_type must be 2 or inf, got {norm_type}")
    return t == float("inf")
