"""Operator schemas for the hot path (namespace ``bitsandbytes::``).

The schema strings are the interface HF Transformers / torch.compile trace, so they are
the reference's (reference bitsandbytes/_ops.py:9-406) verbatim; everything else here is
ours: one table drives the definitions, and the shape functions ("fake" kernels) are
written once per op below.  The optimizer ops (:409-510) are SURVEY.md section 8 row f-4.

The only device with kernels is CUDA (``backends/cuda.py``): the reference's
cpu/default/triton/xpu/mps/hpu fan-out collapses to the single sm_90a path and there is
no CPU fallback -- calling an op on a CPU tensor raises NotImplementedError from the
dispatcher.
"""
from __future__ import annotations

from math import prod
from typing import Optional, Sequence

import torch

NS = "bitsandbytes"

SCHEMAS = {
    "int8_mixed_scaled_mm": "(Tensor A, Tensor CA, Tensor CB, Tensor SCA, Tensor SCB, Tensor? outlier_cols=None, Tensor? bias=None) -> (Tensor, Tensor?)",
    "int8_scaled_mm": "(Tensor A, Tensor B, Tensor row_stats, Tensor col_stats, Tensor? bias=None, ScalarType? dtype=None) -> Tensor",
    "int8_linear_matmul": "(Tensor A, Tensor B) -> Tensor",
    "int8_linear_matmul.out": "(Tensor A, Tensor B, Tensor! out) -> ()",
    "int8_vectorwise_quant": "(Tensor A, float threshold=0.0) -> (Tensor, Tensor, Tensor?)",
    "int8_vectorwise_dequant": "(Tensor A, Tensor stats) -> Tensor",
    "int8_mm_dequant": "(Tensor A, Tensor row_stats, Tensor col_stats, ScalarType? dtype=None, Tensor? bias=None) -> Tensor",
    "int8_double_quant": "(Tensor A, float threshold=0.0) -> (Tensor, Tensor, Tensor, Tensor, Tensor?)",
    "dequantize_4bit": "(Tensor A, Tensor absmax, int blocksize, str quant_type, int[] shape, ScalarType dtype) -> Tensor",
    "dequantize_4bit.out": "(Tensor A, Tensor absmax, int blocksize, str quant_type, int[] shape, ScalarType dtype, Tensor! out) -> ()",
    "quantize_4bit": "(Tensor A, int blocksize, str quant_type, ScalarType quant_storage) -> (Tensor, Tensor)",
    "gemm_4bit": "(Tensor A, Tensor B, int[] shapeB, Tensor absmax, int blocksize, str quant_type, "
    "Tensor? bias=None, Tensor? absmax_8bit=None, Tensor? absmax_code=None, Tensor? absmax_offset=None) -> Tensor",
    "dequantize_blockwise": "(Tensor A, Tensor absmax, Tensor code, int blocksize, ScalarType dtype) -> Tensor",
    "dequantize_blockwise.out": "(Tensor A, Tensor absmax, Tensor code, int blocksize, ScalarType dtype, Tensor! out) -> ()",
    "quantize_blockwise": "(Tensor A, Tensor code, int blocksize) -> (Tensor, Tensor)",
    "gemv_4bit": "(Tensor A, Tensor B, int[] shapeB, Tensor absmax, Tensor code, int blocksize) -> Tensor",
    "gemv_4bit.out": "(Tensor A, Tensor B, int[] shapeB, Tensor absmax, Tensor code, int blocksize, Tensor! out) -> ()",
    "optimizer_update_32bit": "(str optimizer_name, Tensor(a0!) g, Tensor(a1!) p, Tensor(a2!) state1, Tensor(a3!)? state2, "
    "Tensor(a4!)? unorm_vec, float max_unorm, float param_norm, float beta1, float beta2, float beta3, float alpha, "
    "float eps, float weight_decay, int step, float lr, float gnorm_scale, bool skip_zeros=False) -> ()",
    "optimizer_update_8bit_blockwise": "(str optimizer_name, Tensor(a0!) g, Tensor(a1!) p, Tensor(a2!) state1, "
    "Tensor(a3!)? state2, float beta1, float beta2, float beta3, float alpha, float eps, int step, float lr, "
    "Tensor(a4!) qmap1, Tensor(a5!)? qmap2, Tensor(a6!) absmax1, Tensor(a7!)? absmax2, float weight_decay, "
    "float gnorm_scale, bool skip_zeros=False) -> ()",
}

_defined = False


def define_all() -> None:
    """Idempotent: a second import (or a co-installed reference package) must not redefine."""
    global _defined
    if _defined:
        return
    for name, schema in SCHEMAS.items():
        base, _, overload = name.partition(".")
        try:
            torch.library.define(f"{NS}::{name}", schema)
        except RuntimeError as e:  # already defined by another copy of the package in this process
            if "already" not in str(e) and "duplicate" not in str(e).lower():
                raise
    _defined = True


define_all()


def fake(name: str):
    return torch.library.register_fake(f"{NS}::{name}")


def kernel(name: str, device: str = "cuda"):
    return torch.library.register_kernel(f"{NS}::{name}", device)


_4BIT_STORAGE = (torch.uint8, torch.bfloat16, torch.float16, torch.float32)
_FLOATS = (torch.float16, torch.bfloat16, torch.float32)


# ------------------------------------------------------------------------------ shape functions
@fake("int8_mixed_scaled_mm")
def _(A, CA, CB, SCA, SCB, outlier_cols=None, bias=None):
    out = torch.empty((*CA.shape[:-1], CB.shape[0]), device=A.device, dtype=A.dtype)
    n_out = torch.library.get_ctx().new_dynamic_size()
    return out, A.new_empty(n_out, dtype=torch.int64)


@fake("int8_scaled_mm")
def _(A, B, row_stats, col_stats, bias=None, dtype=None):
    return torch.empty((*A.shape[:-1], B.shape[0]), device=A.device, dtype=dtype or torch.float16)


@fake("int8_linear_matmul")
def _(A, B):
    torch._check(A.dtype == torch.int8, lambda: "A must be int8")
    torch._check(B.dtype == torch.int8, lambda: "B must be int8")
    return torch.empty((*A.shape[:-1], B.shape[0]), device=A.device, dtype=torch.int32)


@fake("int8_linear_matmul.out")
def _(A, B, out):
    torch._check(A.dtype == torch.int8, lambda: "A must be int8")
    torch._check(B.dtype == torch.int8, lambda: "B must be int8")
    torch._check(out.shape == (*A.shape[:-1], B.shape[0]), lambda: "out has the wrong shape")
    torch._check(out.dtype == torch.int32, lambda: "out must be int32")


@fake("int8_vectorwise_quant")
def _(A, threshold=0.0):
    q = torch.empty(A.shape, device=A.device, dtype=torch.int8)
    stats = torch.empty(prod(A.shape[:-1]), device=A.device, dtype=torch.float32)
    if threshold == 0.0:
        return q, stats, None
    return q, stats, A.new_empty(torch.library.get_ctx().new_dynamic_size(), dtype=torch.int64)


@fake("int8_vectorwise_dequant")
def _(A, stats):
    torch._check(A.dtype == torch.int8, lambda: "A must be int8")
    return torch.empty_like(A, dtype=torch.float32)


@fake("int8_mm_dequant")
def _(A, row_stats, col_stats, dtype=None, bias=None):
    torch._check(A.dtype == torch.int32, lambda: "A must be int32")
    return torch.empty_like(A, dtype=dtype or torch.float16)


@fake("int8_double_quant")
def _(A, threshold=0.0):
    q_row = torch.empty_like(A, dtype=torch.int8)
    q_col = torch.empty_like(A, dtype=torch.int8)
    row_stats = torch.empty(prod(A.shape[:-1]), device=A.device, dtype=torch.float32)
    col_stats = torch.empty(A.shape[-1], device=A.device, dtype=torch.float32)
    oc = A.new_empty(torch.library.get_ctx().new_dynamic_size(), dtype=torch.int64)
    return q_row, q_col, row_stats, col_stats, oc


def _check_4bit_common(blocksize, quant_type):
    torch._check(quant_type in ("fp4", "nf4"), lambda: f"quant_type must be nf4 or fp4, got {quant_type}")
    torch._check(blocksize >= 0, lambda: "blocksize must be non-negative")


@fake("dequantize_4bit")
def _(A, absmax, blocksize, quant_type, shape, dtype):
    _check_4bit_common(blocksize, quant_type)
    return torch.empty(shape, dtype=dtype, device=A.device)


@fake("dequantize_4bit.out")
def _(A, absmax, blocksize, quant_type, shape, dtype, out):
    _check_4bit_common(blocksize, quant_type)
    torch._check(out.shape == tuple(shape), lambda: f"expected out.shape == {shape}, got {out.shape}")
    torch._check(out.dtype == dtype, lambda: f"expected out.dtype == {dtype}, got {out.dtype}")


@fake("quantize_4bit")
def _(A, blocksize, quant_type, quant_storage):
    _check_4bit_common(blocksize, quant_type)
    n = A.numel()
    absmax = torch.empty((-(n // -blocksize),), device=A.device, dtype=torch.float32)
    out = torch.empty(((n + 1) // (quant_storage.itemsize * 2), 1), device=A.device, dtype=quant_storage)
    return out, absmax


@fake("gemm_4bit")
def _(A, B, shapeB, absmax, blocksize, quant_type, bias=None, absmax_8bit=None, absmax_code=None, absmax_offset=None):
    _check_4bit_common(blocksize, quant_type)
    torch._check(A.dtype in _FLOATS, lambda: f"A must be float16, bfloat16 or float32, got {A.dtype}")
    torch._check(B.dtype in _4BIT_STORAGE, lambda: f"unsupported 4-bit storage dtype {B.dtype}")
    return torch.empty((*A.shape[:-1], shapeB[0]), device=A.device, dtype=A.dtype)


@fake("dequantize_blockwise")
def _(A, absmax, code, blocksize, dtype):
    torch._check(blocksize >= 0, lambda: "blocksize must be non-negative")
    torch._check(A.dtype == torch.uint8, lambda: f"A must be uint8, got {A.dtype}")
    return torch.empty_like(A, dtype=dtype)


@fake("dequantize_blockwise.out")
def _(A, absmax, code, blocksize, dtype, out):
    torch._check(blocksize >= 0, lambda: "blocksize must be non-negative")
    torch._check(A.dtype == torch.uint8, lambda: f"A must be uint8, got {A.dtype}")
    torch._check(out.shape == A.shape, lambda: f"expected out.shape == {A.shape}, got {out.shape}")
    torch._check(out.dtype == dtype, lambda: f"expected out.dtype == {dtype}, got {out.dtype}")


@fake("quantize_blockwise")
def _(A, code, blocksize):
    torch._check(blocksize >= 0, lambda: "blocksize must be non-negative")
    n = A.numel()
    return (torch.empty_like(A, dtype=torch.uint8),
            torch.empty((-(n // -blocksize),), device=A.device, dtype=torch.float32))


def _check_gemv(A, B, shapeB):
    torch._check(A.numel() == A.size(-1), lambda: f"A must be a vector with leading dims of 1, got {A.shape}")
    torch._check(A.dtype in _FLOATS, lambda: f"A must be float16, bfloat16 or float32, got {A.dtype}")
    torch._check(B.dtype in _4BIT_STORAGE, lambda: f"unsupported 4-bit storage dtype {B.dtype}")


@fake("gemv_4bit")
def _(A, B, shapeB, absmax, code, blocksize):
    torch._check(blocksize >= 0, lambda: "blocksize must be non-negative")
    _check_gemv(A, B, shapeB)
    return torch.empty((*A.shape[:-1], shapeB[0]), device=A.device, dtype=A.dtype)


@fake("gemv_4bit.out")
def _(A, B, shapeB, absmax, code, blocksize, out):
    torch._check(blocksize >= 0, lambda: "blocksize must be non-negative")
    _check_gemv(A, B, shapeB)
    torch._check(out.shape == (*A.shape[:-1], shapeB[0]), lambda: "out has the wrong shape")
    torch._check(out.dtype == A.dtype, lambda: "out must have A's dtype")


# ------------------------------------------------------------------------------ device-agnostic glue
# The reference registers this one for every device in pure torch (reference _ops.py:108-121):
# there is no native kernel to replace.
@torch.library.register_kernel(f"{NS}::int8_vectorwise_dequant", None)
def _(A: torch.Tensor, stats: torch.Tensor) -> torch.Tensor:
    # 1/127 as the reference spells it
    return A * stats.view(-1, 1) * 7.874015718698502e-3


def _check_optimizer_args(g, p, state1, state2, state_dtype):
    torch._check(g.numel() == p.numel(), lambda: f"g and p must have the same number of elements, got {g.numel()} and {p.numel()}")
    torch._check(g.dtype in _FLOATS, lambda: f"g must be bfloat16, float16, or float32, got {g.dtype}")
    torch._check(g.dtype == p.dtype, lambda: f"Expected all tensors to have the same dtype, got g.dtype={g.dtype}, p.dtype={p.dtype}")
    torch._check(state1.dtype == state_dtype, lambda: f"state1 must be {state_dtype}, got {state1.dtype}")
    if state2 is not None:
        torch._check(state2.dtype == state_dtype, lambda: f"state2 must be {state_dtype}, got {state2.dtype}")


@fake("optimizer_update_32bit")
def _(optimizer_name, g, p, state1, state2, unorm_vec, max_unorm, param_norm, beta1, beta2, beta3, alpha, eps,
      weight_decay, step, lr, gnorm_scale, skip_zeros=False):
    _check_optimizer_args(g, p, state1, state2, torch.float32)


@fake("optimizer_update_8bit_blockwise")
def _(optimizer_name, g, p, state1, state2, beta1, beta2, beta3, alpha, eps, step, lr, qmap1, qmap2, absmax1, absmax2,
      weight_decay, gnorm_scale, skip_zeros=False):
    _check_optimizer_args(g, p, state1, state2, torch.uint8)
    torch._check(qmap1.dtype == absmax1.dtype == torch.float32,
                 lambda: f"Expected qmap1 and absmax1 to be float32, got {qmap1.dtype}, {absmax1.dtype}")
