"""``bnb.matmul_4bit`` / ``bnb.matmul`` -- routing between the modules and the fused ops.

Same contract as the reference's ``bitsandbytes/autograd/_functions.py`` (MatmulLtState
:57-98, MatMul8bitLt :101-242, MatMul4Bit :300-386, matmul :389-404, matmul_4bit :407-491).
Forward paths run the sm_90a kernels; the backward formulas are the reference's
(grad_A = grad_out . dequant(W); the int8 weight-gradient path uses int8_double_quant).
The CPU/XPU-only ``MatMul8bitFp`` of the reference is not provided.
"""
from __future__ import annotations

import logging
import warnings
from dataclasses import dataclass
from math import prod
from typing import Optional
from warnings import warn

import torch

from .. import functional as F

logger = logging.getLogger(__name__)


def _is_compiling() -> bool:
    return torch.compiler.is_compiling()


class GlobalOutlierPooler:
    """Collects outlier column indices across layers (API compatibility with the reference)."""

    _instance = None

    def __init__(self):
        raise RuntimeError("Call get_instance() instead")

    @classmethod
    def get_instance(cls):
        if cls._instance is None:
            inst = cls.__new__(cls)
            inst.outliers = set()
            inst.model_dim = None
            cls._instance = inst
        return cls._instance

    def add_outliers(self, outlier_idx, feature_dim):
        if self.model_dim is None:
            self.model_dim = feature_dim
        if feature_dim != self.model_dim:
            return  # only the hidden dimension is pooled
        self.outliers.update(outlier_idx.tolist())

    def get_current_outlier_idx(self):
        return torch.Tensor(list(self.outliers)).to(torch.int64)


@dataclass
class MatmulLtState:
    force_no_igemmlt: bool = False
    CB: Optional[torch.Tensor] = None   # int8 weights [N, K]
    SB: Optional[torch.Tensor] = None
    SCB: Optional[torch.Tensor] = None  # fp32 row absmax of the weights [N]
    SBt: Optional[torch.Tensor] = None
    CBt: Optional[torch.Tensor] = None
    subB: Optional[torch.Tensor] = None
    outlier_pool: Optional[GlobalOutlierPooler] = None
    has_accumulated_gradients = False
    threshold = 0.0
    idx: Optional[torch.Tensor] = None
    is_training = True
    has_fp16_weights = True
    use_pool = False

    _deprecated_fields = frozenset({"CxB", "CxBt", "formatB", "_tile_indices"})

    def __getattr__(self, name):
        if name in MatmulLtState._deprecated_fields:
            warnings.warn(f"MatmulLtState.{name} is deprecated and will be removed in the next bitsandbytes release.",
                          FutureWarning, stacklevel=2)
            return None
        raise AttributeError(f"'{type(self).__name__}' object has no attribute '{name}'")

    def reset_grads(self):
        self.CB = self.SB = self.SCB = None
        self.SBt = self.CBt = None


def _empty_result(A, rows_if_match, shape_a, shape_b):
    if A.shape[-1] == shape_a:
        return torch.empty(A.shape[:-1] + shape_b[1:], dtype=A.dtype, device=A.device)
    return torch.empty(A.shape[:-1] + shape_b[:1], dtype=A.dtype, device=A.device)


class MatMul8bitLt(torch.autograd.Function):
    @staticmethod
    def forward(ctx, A, B, out=None, bias=None, state: Optional[MatmulLtState] = None):
        state = state or MatmulLtState()
        ctx.is_empty = False
        if prod(A.shape) == 0:
            ctx.is_empty = True
            ctx.A, ctx.B, ctx.bias = A, B, bias
            return _empty_result(A, None, B.shape[0], B.shape)

        input_shape = A.shape
        if A.dtype != torch.float16 and not _is_compiling():
            logger.warning("MatMul8bitLt: inputs will be cast from %s to float16 during quantization", A.dtype)
        if A.dim() == 3:
            A = A.reshape(-1, A.shape[-1])

        # 1. quantise the activations row-wise (outliers are zeroed in CA as a side effect)
        if ctx.needs_input_grad[1]:
            CA, CAt, SCA, SCAt, outlier_cols = F.int8_double_quant(A.to(torch.float16), threshold=state.threshold)
        else:
            CA, SCA, outlier_cols = F.int8_vectorwise_quant(A.to(torch.float16), threshold=state.threshold)
            CAt = SCAt = None

        # 2. (training with fp16 master weights) quantise the weights
        if state.has_fp16_weights or state.CB is None:
            has_grad = getattr(B, "grad", None) is not None
            if not B.is_contiguous() and B.shape[0] == B.stride(1):
                B = B.contiguous()
            if (state.is_training and not has_grad) or state.CB is None or state.SCB is None:
                state.reset_grads()
                state.CB, state.SCB, _ = F.int8_vectorwise_quant(B.to(torch.float16))

        # 3. int8 GEMM + dequant (+ the outlier columns in 16-bit when threshold > 0)
        if state.threshold > 0.0:
            state.idx = outlier_cols
            output, subA = torch.ops.bitsandbytes.int8_mixed_scaled_mm(A, CA, state.CB, SCA, state.SCB, outlier_cols,
                                                                      bias)
        else:
            output = torch.ops.bitsandbytes.int8_scaled_mm.default(CA, state.CB, SCA, state.SCB, bias=bias,
                                                                   dtype=A.dtype)
            subA = None

        ctx.state = state
        ctx.grad_shape = input_shape
        ctx.dtype_A = A.dtype
        ctx.dtype_bias = None if bias is None else bias.dtype
        if any(ctx.needs_input_grad[:2]):
            ctx.tensors = (CAt, subA, A)
            ctx.tensor_states = (SCAt, state.idx)
        else:
            ctx.tensors = [None, None, None]
            ctx.tensor_states = (None, None)
            ctx.save_for_backward(None, None)

        if len(input_shape) == 3:
            return output.reshape(*input_shape[:-1], state.CB.shape[0])
        return output

    @staticmethod
    def backward(ctx, grad_output):
        if ctx.is_empty:
            bias_grad = None if ctx.bias is None else torch.zeros_like(ctx.bias)
            return torch.zeros_like(ctx.A), torch.zeros_like(ctx.B), None, bias_grad, None

        need_A, need_B, _, need_bias, _ = ctx.needs_input_grad
        CAt, subA, _A = ctx.tensors
        SCAt, idx = ctx.tensor_states
        state: MatmulLtState = ctx.state
        grad_A = grad_B = grad_bias = None

        if need_bias:
            grad_bias = grad_output.sum(0, dtype=ctx.dtype_bias)
        if grad_output.dim() == 3:
            grad_output = grad_output.reshape(-1, grad_output.shape[-1]).contiguous()

        if need_B:
            Cgrad, _, _, SCgradt, _ = F.int8_double_quant(grad_output.to(torch.float16))
            grad_B = torch.ops.bitsandbytes.int8_scaled_mm.default(Cgrad.t().contiguous(), CAt.t(), SCgradt, SCAt,
                                                                   dtype=torch.float16)
            if state.threshold > 0.0 and subA is not None and subA.numel() > 0:
                grad_B[:, idx] += torch.matmul(grad_output.t(), subA)

        if need_A:
            if state.CB is None:
                raise Exception("State must contain CB matrix for backward")
            W = state.CB.to(ctx.dtype_A, copy=True).mul_(state.SCB.unsqueeze(1).mul(1.0 / 127.0))
            grad_A = torch.matmul(grad_output.to(ctx.dtype_A), W).view(ctx.grad_shape)

        return grad_A, grad_B, None, grad_bias, None


def _gemm_4bit(A, B, quant_state, bias):
    """Dispatch to the fused op with plain or double-quantised statistics."""
    if not quant_state.nested:
        return torch.ops.bitsandbytes.gemm_4bit.default(A, B, quant_state.shape, quant_state.absmax,
                                                        quant_state.blocksize, quant_state.quant_type, bias=bias)
    if quant_state.state2.blocksize != 256:
        raise NotImplementedError("nested quantization with state2.blocksize != 256 is not supported")
    return torch.ops.bitsandbytes.gemm_4bit.default(
        A, B, quant_state.shape, quant_state.state2.absmax, quant_state.blocksize, quant_state.quant_type, bias=bias,
        absmax_8bit=quant_state.absmax, absmax_code=quant_state.state2.code, absmax_offset=quant_state.offset)


class MatMul4Bit(torch.autograd.Function):
    @staticmethod
    def forward(ctx, A, B, out=None, bias=None, quant_state: Optional[F.QuantState] = None):
        ctx.is_empty = False
        if A.numel() == 0:
            ctx.is_empty = True
            ctx.A, ctx.B, ctx.bias = A, B, bias
            return _empty_result(A, None, quant_state.shape[0], quant_state.shape)

        B = B.view(-1, 1)  # canonical packed layout; quant_state.shape carries [N, K]
        output = _gemm_4bit(A, B, quant_state, bias)
        if out is not None:
            out.copy_(output)
            output = out

        ctx.state = quant_state
        ctx.dtype_A, ctx.dtype_B = A.dtype, B.dtype
        ctx.dtype_bias = None if bias is None else bias.dtype
        ctx.tensors = (None, B) if any(ctx.needs_input_grad[:2]) else (None, None)
        return output

    @staticmethod
    def backward(ctx, grad_output):
        if ctx.is_empty:
            bias_grad = None if ctx.bias is None else torch.zeros_like(ctx.bias)
            return torch.zeros_like(ctx.A), torch.zeros_like(ctx.B), None, bias_grad, None
        need_A, _, _, need_bias, _ = ctx.needs_input_grad
        _, B = ctx.tensors
        grad_A = grad_bias = None
        if need_bias:
            grad_bias = grad_output.sum(0, dtype=ctx.dtype_bias)
        if need_A:
            # dequantize returns [N, K]: grad_A[M, K] = grad_out[M, N] . W[N, K]
            grad_A = torch.matmul(grad_output, F.dequantize_4bit(B, ctx.state).to(grad_output.dtype))
        return grad_A, None, None, grad_bias, None


def matmul(A, B, out=None, state: Optional[MatmulLtState] = None, threshold=0.0, bias=None):
    state = state or MatmulLtState()
    if threshold > 0.0:
        state.threshold = threshold
    return MatMul8bitLt.apply(A, B, out, bias, state)


def matmul_4bit(A, B, quant_state: F.QuantState, out=None, bias=None):
    if quant_state is None:
        raise ValueError("quant_state is required")
    if len(quant_state.shape) != 2:
        raise ValueError("matmul_4bit: quant_state.shape must be 2D [N, K]")

    B = B.view(-1, 1)
    K = A.shape[-1]

    # Weight quantised from a [K, N] tensor (legacy): dequantize and use the plain linear.
    if K == quant_state.shape[0] and K != quant_state.shape[1]:
        if not _is_compiling():
            warn(f"matmul_4bit: weight was quantized from a [K, N] tensor (quant_state.shape="
                 f"{list(quant_state.shape)}). Re-quantize from the weight in [N, K] (out_features, in_features) "
                 "orientation. This will be an error in a future version.", DeprecationWarning, stacklevel=2)
        W = F.dequantize_4bit(B, quant_state).to(A.dtype)
        result = torch.nn.functional.linear(A, W.t(), bias)
        if out is not None:
            out.copy_(result)
            return out
        return result

    needs_grad = torch.is_grad_enabled() and (A.requires_grad or (bias is not None and bias.requires_grad))
    if needs_grad:
        return MatMul4Bit.apply(A, B, out, bias, quant_state)

    if A.numel() == 0:
        if out is not None:
            return out
        return torch.empty((*A.shape[:-1], quant_state.shape[0]), dtype=A.dtype, device=A.device)
    result = _gemm_4bit(A, B, quant_state, bias)
    if out is not None:
        out.copy_(result)
        return out
    return result
