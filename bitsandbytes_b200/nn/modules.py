"""``bnb.nn`` for the hot path: Linear4bit / LinearNF4 / LinearFP4 / Params4bit and
Linear8bitLt / Int8Params.

Contract of the reference's ``bitsandbytes/nn/modules.py`` (Params4bit :213-484,
fix_4bit_weight_quant_state_from_module :487-501, Linear4bit :504-637, Int8Params :719-809,
maybe_rearrange_weight :812-830, Linear8bitLt :1018-1194): weights are quantised the first
time the module is moved to a device, the packed bytes live in ``weight.data`` (optionally
viewed as ``quant_storage`` so FSDP can flat-shard them), the QuantState rides on the
parameter and is mirrored on the module, and the state_dict keys are the reference's.
Embedding variants, OutlierAwareLinear and the CPU repacking paths are outside the hot path.
"""
from __future__ import annotations

import copy
import logging
from typing import Any, Optional

import torch
from torch import nn

from .. import functional as F
from ..autograd._functions import MatmulLtState, grouped_matmul_4bit, grouped_matmul_8bit, matmul, matmul_4bit
from ..functional import QuantState

logger = logging.getLogger(__name__)

_PARAMS4_FIELDS = ("blocksize", "compress_statistics", "quant_type", "quant_state", "quant_storage", "bnb_quantized",
                   "module")


def _qs_attr(name: str, nested: bool = False, target: Optional[str] = None):
    """Read-only proxy onto the parameter's QuantState.  FSDP's state_dict traversal resolves
    ``weight.absmax`` etc. with getattr; properties (unlike __getattr__) do not break
    torch.compile on Tensor subclasses."""
    field = target or name

    def getter(self):
        qs = self.__dict__.get("quant_state")
        if qs is not None:
            src = qs.state2 if nested else qs
            if src is not None:
                return getattr(src, field)
        raise AttributeError(f"'{type(self).__name__}' object has no attribute '{name}'")

    return property(getter)


class Params4bit(torch.nn.Parameter):
    """Parameter holding packed 4-bit codes; quantises itself on the first move to a device."""

    def __new__(cls, data: Optional[torch.Tensor] = None, requires_grad=False, quant_state: Optional[QuantState] = None,
                blocksize: Optional[int] = None, compress_statistics: bool = True, quant_type: str = "fp4",
                quant_storage: torch.dtype = torch.uint8, module: Optional["Linear4bit"] = None,
                bnb_quantized: bool = False, **kwargs) -> "Params4bit":
        if data is None:
            data = torch.empty(0)
        self = torch.Tensor._make_subclass(cls, data, requires_grad)
        self.blocksize = 64 if blocksize is None else blocksize
        self.compress_statistics = compress_statistics
        self.quant_type = quant_type
        self.quant_state = quant_state
        self.quant_storage = quant_storage
        self.bnb_quantized = bnb_quantized
        self.data = data
        self.module = module
        return self

    absmax = _qs_attr("absmax")
    code = _qs_attr("code")
    quant_map = _qs_attr("quant_map", target="code")
    offset = _qs_attr("offset")
    state2 = _qs_attr("state2")
    nested_offset = _qs_attr("nested_offset", target="offset")
    nested_absmax = _qs_attr("nested_absmax", nested=True, target="absmax")
    nested_blocksize = _qs_attr("nested_blocksize", nested=True, target="blocksize")
    nested_quant_map = _qs_attr("nested_quant_map", nested=True, target="code")
    nested_dtype = _qs_attr("nested_dtype", nested=True, target="dtype")

    # ------------------------------------------------------------------ pickling / copying
    def __getstate__(self):
        state = self.__dict__.copy()
        state["data"] = self.data
        state["requires_grad"] = self.requires_grad
        return state

    def __setstate__(self, state):
        self.requires_grad = state["requires_grad"]
        for k in _PARAMS4_FIELDS:
            setattr(self, k, state[k])
        self.data = state["data"]

    def __deepcopy__(self, memo):
        new = type(self).__new__(type(self))
        state = self.__getstate__()
        new.__setstate__(state)
        new.quant_state = copy.deepcopy(state["quant_state"])
        new.data = copy.deepcopy(state["data"])
        return new

    def __copy__(self):
        new = type(self).__new__(type(self))
        new.__setstate__(self.__getstate__())
        return new

    # ------------------------------------------------------------------ construction from a checkpoint
    @classmethod
    def from_prequantized(cls, data: torch.Tensor, quantized_stats: dict[str, Any], requires_grad: bool = False,
                          device="cuda", module: Optional["Linear4bit"] = None, **kwargs) -> "Params4bit":
        self = torch.Tensor._make_subclass(cls, data.to(device))
        self.requires_grad = requires_grad
        self.quant_state = QuantState.from_dict(qs_dict=quantized_stats, device=device)
        self.blocksize = self.quant_state.blocksize
        self.compress_statistics = self.quant_state.nested
        self.quant_type = self.quant_state.quant_type
        self.bnb_quantized = True
        self.quant_storage = data.dtype
        self.module = module
        if module is not None:
            module.quant_state = self.quant_state
        return self

    # ------------------------------------------------------------------ device movement
    def _quantize(self, device):
        w = self.data.contiguous().to(device)
        packed, state = F.quantize_4bit(w, blocksize=self.blocksize, compress_statistics=self.compress_statistics,
                                        quant_type=self.quant_type, quant_storage=self.quant_storage)
        self.data = packed
        self.quant_state = state
        if self.module is not None:
            self.module.quant_state = state
        self.bnb_quantized = True
        return self

    def cpu(self):
        return self.to(device="cpu")

    def cuda(self, device=None, non_blocking: bool = False):
        return self.to(device="cuda" if device is None else device, non_blocking=non_blocking)

    def to(self, *args, **kwargs):
        device, dtype, non_blocking, _ = torch._C._nn._parse_to(*args, **kwargs)
        # quantisation happens on the first move to a CUDA device: this package has no CPU kernels, so a move of
        # not-yet-quantised weights to the CPU (or a dtype-only .to()) keeps them as they are
        if device is not None and device.type == "cuda" and not self.bnb_quantized:
            return self._quantize(device)
        if self.quant_state is not None:
            self.quant_state.to(device)
        return Params4bit(super().to(device=device, dtype=dtype, non_blocking=non_blocking),
                          requires_grad=self.requires_grad, quant_state=self.quant_state, blocksize=self.blocksize,
                          compress_statistics=self.compress_statistics, quant_type=self.quant_type,
                          quant_storage=self.quant_storage, bnb_quantized=self.bnb_quantized)

    # torch.chunk / torch.split must hand back Params4bit shards (FSDP / tensor-parallel splitting)
    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        result = super().__torch_function__(func, types, args, kwargs)
        if func not in (torch.chunk, torch.split):
            return result
        src = args[0]

        def rewrap(t):
            return cls(data=t, requires_grad=src.requires_grad, quant_state=src.quant_state, blocksize=src.blocksize,
                       compress_statistics=src.compress_statistics, quant_type=src.quant_type,
                       quant_storage=src.quant_storage, module=src.module, bnb_quantized=src.bnb_quantized)

        return tuple(rewrap(t) for t in result) if isinstance(result, tuple) else rewrap(result)


def fix_4bit_weight_quant_state_from_module(module: "Linear4bit"):
    """FSDP and friends replace the parameter object and lose ``weight.quant_state``; the module
    keeps a mirror from which it is restored."""
    if getattr(module.weight, "quant_state", None) is not None:
        return
    if getattr(module, "quant_state", None) is None:
        logger.warning("FP4 quantization state not initialized. Please call .cuda() or .to(device) on the "
                       "LinearFP4 layer first.")
    if module.weight.shape[1] != 1:
        raise AssertionError("expected the packed weight in [n_bytes, 1] layout")
    if not isinstance(module.weight, Params4bit):
        module.weight = Params4bit(module.weight, quant_storage=module.quant_storage, bnb_quantized=True)
    module.weight.quant_state = module.quant_state


class Linear4bit(nn.Linear):
    """QLoRA-style 4-bit linear layer.  ``module.to("cuda")`` quantises the loaded 16/32-bit
    weights; ``forward`` runs the fused dequant-GEMM (wgmma on H100)."""

    def __init__(self, input_features, output_features, bias=True, compute_dtype=None, compress_statistics=True,
                 quant_type="fp4", quant_storage=torch.uint8, device=None):
        super().__init__(input_features, output_features, bias, device)
        self.weight = Params4bit(self.weight.data, requires_grad=False, compress_statistics=compress_statistics,
                                 quant_type=quant_type, quant_storage=quant_storage, module=self)
        self.compute_dtype = compute_dtype
        self.compute_type_is_set = compute_dtype is not None
        self.quant_state = None
        self.quant_storage = quant_storage
        self.support_avx512bf16_for_cpu = False  # attribute probed by downstream code; no CPU path here

    def set_compute_type(self, x):
        if x.dtype in (torch.float32, torch.bfloat16):
            self.compute_dtype = x.dtype  # safe and fast to compute in the input dtype
        elif x.dtype == torch.float16 and self.compute_dtype in (None, torch.float32):
            single = x.numel() == x.shape[-1]
            logger.warning("Input type into Linear4bit is torch.float16, but bnb_4bit_compute_dtype=torch.float32 "
                           "(default). This will lead to slow inference%s.", "" if single else " or training speed")

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)
        _save_quant_state(self, destination, prefix, keep_vars)

    def _compute_inputs(self, x: torch.Tensor):
        """x and the bias in the compute dtype (set from the first input unless given)."""
        if not self.compute_type_is_set:
            self.set_compute_type(x)
            self.compute_type_is_set = True
        if self.compute_dtype is not None:
            x = x.to(self.compute_dtype)
        bias = self.bias
        if bias is not None:
            if bias.dtype != x.dtype:
                bias.data = bias.data.to(x.dtype)
            bias = bias.to(self.compute_dtype)
        return x, bias

    def forward(self, x: torch.Tensor):
        fix_4bit_weight_quant_state_from_module(self)
        quant_state = self.weight.quant_state
        inp_dtype = x.dtype
        x, bias = self._compute_inputs(x)
        return matmul_4bit(x, self.weight, bias=bias, quant_state=quant_state).to(inp_dtype)


def _save_quant_state(module: nn.Module, destination, prefix, keep_vars):
    """The packed QuantState entries of a 4-bit weight next to it in the state dict (``weight.absmax`` ...), from which
    ``Params4bit.from_prequantized`` rebuilds it."""
    qs = getattr(module.weight, "quant_state", None)
    if qs is not None:
        for k, v in qs.as_dict(packed=True).items():
            destination[prefix + "weight." + k] = v if keep_vars else v.detach()


class GroupedLinear4bit(nn.Module):
    """The experts of a mixture-of-experts layer on 4-bit weights: ``num_experts`` linear maps ``in_features ->
    out_features`` stored as one ``[E, N, K]`` expert tensor, quantised as one tensor on the first move to CUDA (as
    ``Linear4bit`` quantises its weight), with an optional ``[E, N]`` bias.  ``forward(x, offs)`` takes the
    expert-sorted rows ``x [M, K]`` and the int32 end row of each expert ``offs [E]`` on the device, and returns
    ``[M, N]``: every expert in one launch of the grouped GEMM (:func:`bitsandbytes_b200.grouped_matmul_4bit`).
    Routing (top-k, sorting, scattering back with the router weights) stays with the model."""

    def __init__(self, num_experts, in_features, out_features, bias=False, compute_dtype=None,
                 compress_statistics=True, quant_type="fp4", quant_storage=torch.uint8, device=None):
        super().__init__()
        self.num_experts, self.in_features, self.out_features = num_experts, in_features, out_features
        w = torch.empty((num_experts, out_features, in_features), device=device)
        nn.init.kaiming_uniform_(w.view(-1, in_features), a=5**0.5)  # each expert initialised as nn.Linear's weight
        self.weight = Params4bit(w, requires_grad=False, compress_statistics=compress_statistics, quant_type=quant_type,
                                 quant_storage=quant_storage, module=self)
        if bias:
            bound = 1 / in_features**0.5 if in_features > 0 else 0
            self.bias = nn.Parameter(torch.empty((num_experts, out_features), device=device).uniform_(-bound, bound))
        else:
            self.register_parameter("bias", None)
        self.compute_dtype = compute_dtype
        self.compute_type_is_set = compute_dtype is not None
        self.quant_state = None
        self.quant_storage = quant_storage

    set_compute_type = Linear4bit.set_compute_type
    _compute_inputs = Linear4bit._compute_inputs

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)
        _save_quant_state(self, destination, prefix, keep_vars)

    def extra_repr(self) -> str:
        return (f"num_experts={self.num_experts}, in_features={self.in_features}, out_features={self.out_features}, "
                f"bias={self.bias is not None}")

    def forward(self, x: torch.Tensor, offs: torch.Tensor):
        fix_4bit_weight_quant_state_from_module(self)
        inp_dtype = x.dtype
        x, bias = self._compute_inputs(x)
        return grouped_matmul_4bit(x, self.weight, self.weight.quant_state, offs, bias=bias).to(inp_dtype)


class LinearFP4(Linear4bit):
    def __init__(self, input_features, output_features, bias=True, compute_dtype=None, compress_statistics=True,
                 quant_storage=torch.uint8, device=None):
        super().__init__(input_features, output_features, bias, compute_dtype, compress_statistics, "fp4",
                         quant_storage, device)


class LinearNF4(Linear4bit):
    def __init__(self, input_features, output_features, bias=True, compute_dtype=None, compress_statistics=True,
                 quant_storage=torch.uint8, device=None):
        super().__init__(input_features, output_features, bias, compute_dtype, compress_statistics, "nf4",
                         quant_storage, device)


# ======================================================================================= LLM.int8()
class Int8Params(torch.nn.Parameter):
    def __new__(cls, data: Optional[torch.Tensor] = None, requires_grad=True, has_fp16_weights=False,
                CB: Optional[torch.Tensor] = None, SCB: Optional[torch.Tensor] = None, **kwargs):
        if data is None:
            data = torch.empty(0)
        obj = torch.Tensor._make_subclass(cls, data, requires_grad)
        obj.CB = CB
        obj.SCB = SCB
        obj.has_fp16_weights = has_fp16_weights
        return obj

    def _quantize(self, device):
        if self.has_fp16_weights:
            return super().to(device)
        W = self.data.contiguous().to(device=device, dtype=torch.float16)
        CB, SCB, _ = F.int8_vectorwise_quant(W)  # int8 row-major [N, K] + fp32 row absmax [N]
        self.data = CB
        self.CB = CB
        self.SCB = SCB
        return self

    def cpu(self):
        return self.to(device="cpu")

    def cuda(self, device=None, non_blocking: bool = False):
        return self.to(device="cuda" if device is None else device, non_blocking=non_blocking)

    def __deepcopy__(self, memo):
        return type(self).__new__(type(self), data=copy.deepcopy(self.data, memo), requires_grad=self.requires_grad,
                                  has_fp16_weights=self.has_fp16_weights, CB=copy.deepcopy(self.CB, memo),
                                  SCB=copy.deepcopy(self.SCB, memo))

    def to(self, *args, **kwargs):
        device, dtype, non_blocking, _ = torch._C._nn._parse_to(*args, **kwargs)
        quantized = self.data.dtype == torch.int8
        if not quantized and device is not None and device.type == "cuda" and self.data.device.type == "cpu":
            return self._quantize(device)  # (no CPU kernels: a move to the CPU leaves fp weights unquantised)
        new = Int8Params(super().to(device=device, dtype=dtype, non_blocking=non_blocking),
                         requires_grad=self.requires_grad, has_fp16_weights=self.has_fp16_weights)
        if quantized:
            new.CB = new.data
            if device is not None and self.SCB is not None and self.SCB.device.type != "meta":
                new.SCB = self.SCB.to(device)
        return new


def maybe_rearrange_weight(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
    """Old checkpoints carry a ``weight_format`` entry; only the row-major format (0) exists now."""
    if state_dict.get(f"{prefix}weight") is None:
        return
    fmt = state_dict.pop(f"{prefix}weight_format", "row")
    if isinstance(fmt, torch.Tensor):
        fmt = fmt.item()
    if isinstance(fmt, int):
        if fmt != 0:
            raise ValueError(f"Expected supported weight format - got {fmt}")
        fmt = "row"
    if fmt != "row":
        raise ValueError(f"Only 'row' weight format is supported, got {fmt}")


class Linear8bitLt(nn.Linear):
    """LLM.int8() linear layer: int8 weights (row-wise absmax), activations quantised on the fly,
    columns with outliers (|x| >= threshold) computed in 16-bit."""

    def __init__(self, input_features: int, output_features: int, bias=True, has_fp16_weights=True, threshold=0.0,
                 index=None, device=None):
        super().__init__(input_features, output_features, bias, device)
        self.state = MatmulLtState()
        self.index = index
        self.state.threshold = threshold
        self.state.has_fp16_weights = has_fp16_weights
        if threshold > 0.0 and not has_fp16_weights:
            self.state.use_pool = True
        self.weight = Int8Params(self.weight.data, has_fp16_weights=has_fp16_weights, requires_grad=has_fp16_weights)
        self._register_load_state_dict_pre_hook(maybe_rearrange_weight)

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)
        if self.state.has_fp16_weights:
            return
        # CB is weight.data; only SCB is extra.  It lives on the weight before the first forward
        # and on self.state after it.
        scb = getattr(self.weight, "SCB", None)
        if scb is None:
            scb = self.state.SCB
        if scb is not None:
            destination[prefix + "SCB"] = scb if keep_vars else scb.detach()
            destination[prefix + "weight_format"] = torch.tensor(0, dtype=torch.uint8)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                      error_msgs)
        for key in list(unexpected_keys):
            if key[len(prefix):] != "SCB":
                continue
            scb = getattr(self.weight, "SCB", None)
            if scb is None:
                raise RuntimeError("Loading a quantized checkpoint into non-quantized Linear8bitLt is not supported. "
                                   "Please call module.cuda() before module.load_state_dict()")
            scb.copy_(state_dict[key])
            if self.state.SCB is not None:
                self.state.SCB = self.weight.SCB
            unexpected_keys.remove(key)

    def init_8bit_state(self):
        self.state.CB = self.weight.CB
        self.state.SCB = self.weight.SCB
        self.weight.CB = None
        self.weight.SCB = None

    def to(self, *args, **kwargs):
        result = super().to(*args, **kwargs)
        device, _, _, _ = torch._C._nn._parse_to(*args, **kwargs)
        if device is not None:
            if result.state.CB is not None:
                result.state.CB = result.state.CB.to(device)
            if result.state.SCB is not None:
                result.state.SCB = result.state.SCB.to(device)
        return result

    def forward(self, x: torch.Tensor):
        self.state.is_training = self.training
        if self.weight.CB is not None:
            self.init_8bit_state()
        if self.bias is not None and self.bias.dtype != x.dtype:
            self.bias.data = self.bias.data.to(x.dtype)
        out = matmul(x, self.weight, bias=self.bias, state=self.state)
        if not self.state.has_fp16_weights and self.state.CB is not None:
            self.weight.data = self.state.CB
        return out


class GroupedLinear8bitLt(nn.Module):
    """The experts of a mixture-of-experts layer on LLM.int8() weights: ``num_experts`` linear maps ``in_features ->
    out_features`` stored as one ``[E, N, K]`` expert tensor, quantised row-wise as one tensor on the first move to CUDA
    (as ``Linear8bitLt`` quantises its weight, so expert e's codes and statistics are the ones a ``Linear8bitLt`` of that
    expert holds), with an optional ``[E, N]`` bias.  ``forward(x, offs)`` takes the expert-sorted rows ``x [M, K]`` and
    the int32 end row of each expert ``offs [E]`` on the device, and returns ``[M, N]``: every expert in one GEMM
    launch (:func:`bitsandbytes_b200.grouped_matmul_8bit`), each with its own outlier columns when ``threshold > 0``.
    The state dict has ``Linear8bitLt``'s keys: ``weight`` (the int8 codes), ``SCB`` and ``weight_format``.  Routing
    stays with the model."""

    def __init__(self, num_experts, in_features, out_features, bias=False, threshold=0.0, has_fp16_weights=False,
                 device=None):
        super().__init__()
        if has_fp16_weights:
            raise ValueError("GroupedLinear8bitLt: has_fp16_weights=True is not supported: the expert weights are "
                             "frozen int8 codes")
        self.num_experts, self.in_features, self.out_features = num_experts, in_features, out_features
        self.threshold = threshold
        w = torch.empty((num_experts, out_features, in_features), device=device)
        nn.init.kaiming_uniform_(w.view(-1, in_features), a=5**0.5)  # each expert initialised as nn.Linear's weight
        self.weight = Int8Params(w, requires_grad=False, has_fp16_weights=False)
        if bias:
            bound = 1 / in_features**0.5 if in_features > 0 else 0
            self.bias = nn.Parameter(torch.empty((num_experts, out_features), device=device).uniform_(-bound, bound))
        else:
            self.register_parameter("bias", None)
        self._register_load_state_dict_pre_hook(maybe_rearrange_weight)

    def extra_repr(self) -> str:
        return (f"num_experts={self.num_experts}, in_features={self.in_features}, out_features={self.out_features}, "
                f"bias={self.bias is not None}, threshold={self.threshold}")

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)
        scb = getattr(self.weight, "SCB", None)
        if scb is not None:
            destination[prefix + "SCB"] = scb if keep_vars else scb.detach()
            destination[prefix + "weight_format"] = torch.tensor(0, dtype=torch.uint8)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        w, scb = state_dict.get(prefix + "weight"), state_dict.get(prefix + "SCB")
        if w is None or scb is None or w.dtype != torch.int8:
            super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                          error_msgs)
            return
        # quantised codes: they replace the weight whether or not it has been quantised yet (on CPU they move to the
        # device with the module, as Int8Params does), so a checkpoint loads before or after .cuda()
        own = (prefix + "weight", prefix + "SCB", prefix + "weight_format")
        rest = {k: v for k, v in state_dict.items() if k not in own}
        super()._load_from_state_dict(rest, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)
        for keys in (missing_keys, unexpected_keys):
            keys[:] = [k for k in keys if k not in own]
        shape = (self.num_experts, self.out_features, self.in_features)
        if tuple(w.shape) != shape or tuple(scb.shape) != (shape[0] * shape[1],):
            error_msgs.append(f"size mismatch for {prefix}weight / {prefix}SCB: expected int8 {list(shape)} and "
                              f"[{shape[0] * shape[1]}], got {list(w.shape)} and {list(scb.shape)}")
            return
        dev = self.weight.device
        CB = w.detach().to(dev, copy=True).contiguous()
        self.weight = Int8Params(CB, requires_grad=False, has_fp16_weights=False, CB=CB,
                                 SCB=scb.detach().to(device=dev, dtype=torch.float32, copy=True))

    def forward(self, x: torch.Tensor, offs: torch.Tensor):
        CB = self.weight.data
        if CB.dtype != torch.int8:
            raise RuntimeError("GroupedLinear8bitLt: the weight is not quantised yet: move the module to CUDA first")
        scb = self.weight.SCB
        if scb.device != CB.device:  # a module moved after loading codes on the CPU: the statistics follow the codes
            scb = self.weight.SCB = scb.to(CB.device)
        if self.bias is not None and self.bias.dtype != x.dtype:
            self.bias.data = self.bias.data.to(x.dtype)
        return grouped_matmul_8bit(x, CB, scb, offs, threshold=self.threshold, bias=self.bias)
