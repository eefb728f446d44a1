"""``bnb.matmul_4bit`` / ``bnb.matmul`` -- routing between the modules and the fused ops.

Same contract as the reference's ``bitsandbytes/autograd/_functions.py`` (MatmulLtState
:57-98, MatMul8bitLt :101-242, MatMul4Bit :300-386, matmul :389-404, matmul_4bit :407-491).
Forward paths run the sm_90a kernels and are bit-identical to the reference.  grad_A is the
reference's formula (grad_out . dequant(W)).  The int8 weight gradient of ``MatMul8bitLt``
differs from the reference on purpose, because the reference's value is not the gradient:
it dequantises the *row* codes of grad_out with its *column* statistics, and with
``threshold > 0`` it adds the outlier columns of A twice (once in the int8 product, once from
``subA``).  Here both operands of grad_outᵀ . A are column codes with their column statistics,
and the outlier columns are zeroed in the int8 operand before ``subA`` adds them in full.
With ``threshold > 0``, a forward inside CUDA graph capture keeps the outlier columns on the device
(``_int8_forward_captured``); that route serves inference only and leaves ``state.idx`` as it was.
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
from .._ops import check_int8_grouped
from ..backends.cuda import int8_dequant_rows, int8_mixed_mm_flags, int8_vectorwise_quant_flags, int8_zero_columns

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


def _quantize_weight(B, state: MatmulLtState) -> None:
    """state.CB / state.SCB from the fp16 master weight B, when they are missing or stale."""
    if state.has_fp16_weights or state.CB is None:
        has_grad = getattr(B, "grad", None) is not None
        if not B.is_contiguous() and B.shape[0] == B.stride(1):
            B = B.contiguous()
        if (state.is_training and not has_grad) or state.CB is None or state.SCB is None:
            state.reset_grads()
            state.CB, state.SCB, _ = F.int8_vectorwise_quant(B.to(torch.float16))


_CAPTURED_TRAINING = ("MatMul8bitLt: under CUDA graph capture, LLM.int8() with threshold > 0 runs inference only "
                      "(torch.no_grad(), or no input that requires grad): its backward needs the outlier columns, whose "
                      "number depends on the data")


def _int8_forward_captured(A, B, bias, state: MatmulLtState):
    """LLM.int8() inference forward with threshold > 0 while a CUDA graph is being captured.  The outlier columns and
    their count stay on the device (``int8_mixed_mm_flags``): no host synchronisation, and the captured graph gives the
    eager result for whatever outlier set a replay meets.  ``state.idx`` is not updated on this route, because the
    column list has a data-dependent length."""
    A2 = A.reshape(-1, A.shape[-1])
    CA, SCA, col_flags = int8_vectorwise_quant_flags(A2.to(torch.float16), state.threshold)
    _quantize_weight(B, state)
    out = int8_mixed_mm_flags(A2, CA, state.CB, SCA, state.SCB, col_flags, bias)
    return out.reshape(*A.shape[:-1], state.CB.shape[0])


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

        if state.threshold > 0.0 and A.is_cuda and torch.cuda.is_current_stream_capturing():
            if any(ctx.needs_input_grad):
                raise RuntimeError(_CAPTURED_TRAINING)
            return _int8_forward_captured(A, B, bias, state)

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
        _quantize_weight(B, state)

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
            # grad_B[N, K] = grad_outputᵀ · A, contracted over the tokens: both operands are quantised per column
            # (per output feature / per input feature), so the column codes go with the column statistics.
            _, Cgradt, _, SCgradt, _ = F.int8_double_quant(grad_output.to(torch.float16))
            outliers = state.threshold > 0.0 and subA is not None and subA.numel() > 0
            if outliers:
                # CAt zeroes only the entries >= threshold; subA carries the outlier columns whole, so the rest of
                # those columns must leave the int8 product or it is counted twice
                int8_zero_columns(CAt, idx)
            grad_B = torch.ops.bitsandbytes.int8_scaled_mm.default(Cgradt.t().contiguous(), CAt.t(), SCgradt, SCAt,
                                                                   dtype=torch.float16)
            if outliers:
                # fp32 operands: one rounding, to the fp16 of grad_B, whatever the input dtype
                grad_B[:, idx] += torch.matmul(grad_output.t().float(), subA.float())

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
    # Under no_grad nothing is recorded, but MatMul8bitLt.forward cannot see that: it runs with grad disabled, and
    # ctx.needs_input_grad mirrors requires_grad in every grad mode (True for fp16 master weights).
    if (state.threshold > 0.0 and not torch.is_grad_enabled() and A.is_cuda and A.numel() > 0
            and torch.cuda.is_current_stream_capturing()):
        return _int8_forward_captured(A, B, bias, state)
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


def _gemm_4bit_grouped(A, B, quant_state, offs, bias):
    """The grouped op with plain or double-quantised statistics."""
    if not quant_state.nested:
        return torch.ops.bitsandbytes.gemm_4bit_grouped.default(A, B, quant_state.shape, quant_state.absmax,
                                                                quant_state.blocksize, quant_state.quant_type, offs,
                                                                bias=bias)
    if quant_state.state2.blocksize != 256:
        raise NotImplementedError("nested quantization with state2.blocksize != 256 is not supported")
    return torch.ops.bitsandbytes.gemm_4bit_grouped.default(
        A, B, quant_state.shape, quant_state.state2.absmax, quant_state.blocksize, quant_state.quant_type, offs,
        bias=bias, absmax_8bit=quant_state.absmax, absmax_code=quant_state.state2.code,
        absmax_offset=quant_state.offset)


def _clamped_ends(offs, M):
    """end_e = min(max(offs[e], end_{e-1}), M), end_{-1} = 0: the kernel's clamp of the expert ends, on the device."""
    return offs.clamp(min=0).cummax(0).values.clamp(max=M)


def _grouped_backward(grad_output, offs, E, N, need_A, need_bias, weight):
    """(grad_A, grad_bias) of a grouped expert GEMM with a frozen weight: ``weight()`` gives the dequantised ``[E, N,
    K]`` expert tensor in grad_output's dtype, grad_A is ``grouped_mm`` over the clamped ends with the rows past the
    last end zeroed, and grad_bias the per-expert segment sums of grad_output.  Nothing reads ``offs`` on the host."""
    M = grad_output.shape[0]
    ends = _clamped_ends(offs, M)
    grad_A = grad_bias = None
    if need_A:
        W = weight()  # [E, N, K]
        grad_A = torch.nn.functional.grouped_mm(grad_output.contiguous(), W, offs=ends)
        # rows past the last expert's end belong to no expert: their gradient is zero
        routed = torch.arange(M, device=grad_A.device).unsqueeze(1) < ends[-1]
        grad_A = torch.where(routed, grad_A, torch.zeros((), dtype=grad_A.dtype, device=grad_A.device))
    if need_bias:
        # segment sums of grad_output's rows in fp32; the rows past the last end go to a discarded segment E
        eid = torch.searchsorted(ends, torch.arange(M, device=ends.device, dtype=ends.dtype), right=True)
        sums = torch.zeros((E + 1, N), dtype=torch.float32, device=grad_output.device)
        grad_bias = sums.index_add_(0, eid, grad_output.float())[:E].to(grad_output.dtype)
    return grad_A, grad_bias


class GroupedMatMul4Bit(torch.autograd.Function):
    """The grouped 4-bit GEMM with a frozen weight.  The backward (bf16) dequantises the expert tensor once and runs
    ``grouped_mm`` for grad_A; nothing in either direction reads ``offs`` on the host."""

    @staticmethod
    def forward(ctx, A, B, offs, bias, quant_state):
        out = _gemm_4bit_grouped(A, B, quant_state, offs, bias)
        ctx.state = quant_state
        ctx.save_for_backward(B, offs)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        need_A, _, _, need_bias, _ = ctx.needs_input_grad
        B, offs = ctx.saved_tensors
        E, N, K = ctx.state.shape
        grad_A, grad_bias = _grouped_backward(grad_output, offs, E, N, need_A, need_bias,
                                              lambda: F.dequantize_4bit(B, ctx.state).to(grad_output.dtype))
        return grad_A, None, None, grad_bias, None


def grouped_matmul_4bit(A, B, quant_state: F.QuantState, offs, bias=None):
    """Every expert of a mixture-of-experts layer in one launch, on a 4-bit expert tensor: for the rows of expert e,
    ``offs[e-1] <= m < offs[e]`` of the expert-sorted ``A [M, K]``, ``out[m] = A[m] . W[e]^T + bias[e]``; rows past
    ``offs[E-1]`` are zero.  ``B``/``quant_state`` are the ``[E, N, K]`` weight quantised as one tensor
    (``F.quantize_4bit``, ``Params4bit``), ``offs`` the int32 ``[E]`` end rows on the device (malformed ones are
    clamped on the device), ``bias`` an optional ``[E, N]``.  The weight is frozen; A and the bias train in bf16 only."""
    if quant_state is None:
        raise ValueError("quant_state is required")
    if len(quant_state.shape) != 3:
        raise ValueError(f"grouped_matmul_4bit: quant_state.shape must be the [E, N, K] of the expert tensor, got "
                         f"{list(quant_state.shape)}")
    E, N, K = quant_state.shape
    if A.dim() != 2 or A.shape[1] != K:
        hint = " (the weight was quantised as [E, K, N]: quantise it as [E, N, K])" if A.shape[-1] == N else ""
        raise ValueError(f"grouped_matmul_4bit: A must be [M, {K}] for an [E, N, K] = {list(quant_state.shape)} "
                         f"weight, got {list(A.shape)}{hint}")
    B = B.view(-1, 1)
    needs_grad = torch.is_grad_enabled() and (A.requires_grad or (bias is not None and bias.requires_grad))
    if not needs_grad:
        return _gemm_4bit_grouped(A, B, quant_state, offs, bias)
    if A.dtype != torch.bfloat16:
        raise ValueError(f"grouped_matmul_4bit: training runs in bfloat16 only (the input gradient is "
                         f"torch.nn.functional.grouped_mm), got {A.dtype} with requires_grad")
    if N % 8 != 0:
        raise ValueError(f"grouped_matmul_4bit: training needs N % 8 == 0 (grouped_mm's row stride), got N = {N}")
    return GroupedMatMul4Bit.apply(A, B, offs, bias, quant_state)


class GroupedMatMul8bitLt(torch.autograd.Function):
    """The grouped LLM.int8() GEMM with a frozen weight.  The backward (bf16) takes grad_A through ``grouped_mm`` with
    the whole expert tensor dequantised as ``MatMul8bitLt.backward`` dequantises a weight, ``CB * (SCB / 127)`` with the
    outliers ignored; nothing in either direction reads ``offs`` on the host."""

    @staticmethod
    def forward(ctx, A, CB, SCB, offs, bias, threshold):
        out = torch.ops.bitsandbytes.int8_grouped_mm.default(A, CB, SCB, offs, threshold=threshold, bias=bias)
        ctx.save_for_backward(CB, SCB, offs)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        need_A, _, _, _, need_bias, _ = ctx.needs_input_grad
        CB, SCB, offs = ctx.saved_tensors
        E, N, K = CB.shape
        grad_A, grad_bias = _grouped_backward(
            grad_output, offs, E, N, need_A, need_bias,
            lambda: int8_dequant_rows(CB.reshape(E * N, K), SCB, grad_output.dtype).view(E, N, K))
        return grad_A, None, None, None, grad_bias, None


def grouped_matmul_8bit(A, CB, SCB, offs, threshold=0.0, bias=None):
    """Every expert of a mixture-of-experts layer in one int8 GEMM launch: for the rows of expert e,
    ``offs[e-1] <= m < offs[e]`` of the expert-sorted ``A [M, K]`` (fp16 / bf16), ``out[m]`` is what the inference
    ``Linear8bitLt`` with this ``threshold`` computes on expert e's rows alone -- its own outlier columns included -- and
    rows past ``offs[E-1]`` are zero.  ``CB [E, N, K]`` / ``SCB [E * N]`` are the expert tensor quantised row-wise as one
    tensor (``F.int8_vectorwise_quant``, ``Int8Params``), ``offs`` the int32 ``[E]`` end rows on the device (malformed
    ones are clamped on the device), ``bias`` an optional ``[E, N]``.  The weight is frozen; A and the bias train in
    bf16 only."""
    check_int8_grouped(A, CB, SCB, offs, threshold, bias)
    needs_grad = torch.is_grad_enabled() and (A.requires_grad or (bias is not None and bias.requires_grad))
    if not needs_grad:
        return torch.ops.bitsandbytes.int8_grouped_mm.default(A, CB, SCB, offs, threshold=threshold, bias=bias)
    if A.dtype != torch.bfloat16:
        raise ValueError(f"grouped_matmul_8bit: training runs in bfloat16 only (the input gradient is "
                         f"torch.nn.functional.grouped_mm), got {A.dtype} with requires_grad")
    N = CB.shape[1]
    if N % 8 != 0:
        raise ValueError(f"grouped_matmul_8bit: training needs N % 8 == 0 (grouped_mm's row stride), got N = {N}")
    return GroupedMatMul8bitLt.apply(A, CB, SCB, offs, bias, float(threshold))
