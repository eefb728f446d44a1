"""``bnb.functional`` for the hot path.

Same names, argument meaning and error behaviour as the reference's
``bitsandbytes/functional.py`` (QuantState :420-610, quantize_blockwise :613,
dequantize_blockwise :689, get_4bit_type :772, quantize_4bit :884, dequantize_4bit :992,
gemv_4bit :1300, int8_* :1536-1673, create_dynamic_map :296, optimizer_update_32bit :1080,
optimizer_update_8bit_blockwise :1169, the paged-memory helpers :25-160).  The deprecated igemm family and
the CPU weight-repacking helpers of the reference are not provided.

All tensor work is done by the ``bitsandbytes::`` ops whose only kernels are the sm_90a
ones (``backends/cuda.py``); tensors must live on a CUDA device.
"""
from __future__ import annotations

import ctypes as ct
import itertools
from typing import Any, Optional, Sequence, Union

import torch
from torch import Tensor

from . import _ops  # noqa: F401  (defines the op schemas)
from .backends import cuda as _cuda_backend  # noqa: F401  (registers the CUDA kernels)
from .cextension import lib  # noqa: F401
from .utils import pack_dict_to_tensor, unpack_tensor_to_dict

name2qmap: dict[str, Tensor] = {}

_ops_ns = torch.ops.bitsandbytes

# ------------------------------------------------------------------------------------ code books
_NF4_VALUES = (
    -1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
    -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
    0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941,
    0.7229568362236023, 1.0,
)
# bit 3 = sign, low 3 bits index {0, 0.0625, 8, 12, 4, 6, 2, 3}; normalised by the max (12)
_FP4_MAGNITUDES = (0.0, 0.0625, 8.0, 12.0, 4.0, 6.0, 2.0, 3.0)


def create_dynamic_map(signed: bool = True, max_exponent_bits: int = 7, total_bits: int = 8) -> Tensor:
    """The 8-bit "dynamic" code book (Dettmers 2015, arXiv:1511.04561): a sign bit, a unary
    exponent of up to ``max_exponent_bits`` and a linear fraction in the remaining bits.
    Value-for-value equal to the reference's map (reference functional.py:296-348; pinned by
    tests/test_host_cpu.py against a golden copy)."""
    mantissa_bits_base = total_bits - 1 - max_exponent_bits
    values: list[float] = []
    n_groups = max_exponent_bits
    for e in range(n_groups):
        span = e + mantissa_bits_base
        count = (2**span + 1) if signed else (2 ** (span + 1) + 1)
        edges = torch.linspace(0.1, 1, int(count), dtype=torch.float32)
        centers = (edges[:-1] + edges[1:]) / 2.0
        mag = 10 ** (e - (max_exponent_bits - 1))
        values += (mag * centers).tolist()
        if signed:
            values += (-mag * centers).tolist()
    extra = 2**mantissa_bits_base - 1
    if extra > 0:
        edges = torch.linspace(0.1, 1, extra + 1, dtype=torch.float32)
        centers = (edges[:-1] + edges[1:]) / 2.0
        mag = 10 ** ((n_groups - 1) - (max_exponent_bits - 1))
        values += (mag * centers).tolist()
        if signed:
            values += (-mag * centers).tolist()
    values += [0, 1.0]
    if len(values) != 2**total_bits:
        raise AssertionError(f"dynamic map has {len(values)} entries, expected {2 ** total_bits}")
    values += [0] * (256 - len(values))
    values.sort()
    return torch.tensor(values, dtype=torch.float32)


def create_normal_map(offset: float = 0.9677083, use_extra_value: bool = True) -> Tensor:
    """NormalFloat quantiles (QLoRA); needs scipy.  Used only to regenerate the NF4 table/tree."""
    from scipy.stats import norm

    if use_extra_value:
        pos = norm.ppf(torch.linspace(offset, 0.5, 9)[:-1]).tolist()
        neg = (-norm.ppf(torch.linspace(offset, 0.5, 8)[:-1])).tolist()
        pad = 256 - 15
    else:
        pos = norm.ppf(torch.linspace(offset, 0.5, 8)[:-1]).tolist()
        neg = (-norm.ppf(torch.linspace(offset, 0.5, 8)[:-1])).tolist()
        pad = 256 - 14
    vals = torch.tensor(pos + [0] * pad + neg)
    vals = vals.sort().values
    return vals / vals.max()


def create_linear_map(signed: bool = True, total_bits: int = 8, add_zero: bool = True) -> Tensor:
    """Evenly spaced code book on [-1, 1] (or [0, 1]); fewer than 8 bits are simulated by zero entries
    in the middle of the 256-entry table, and a signed table then gives up one level so that it stays
    centred on zero (reference functional.py:150-166; pinned against a golden copy)."""
    levels = 2**total_bits
    if signed and (add_zero or total_bits < 8):
        levels -= 1
    ramp = torch.linspace(-1.0 if signed else 0.0, 1.0, levels)
    pad = 256 - ramp.numel()
    if pad == 0:
        return ramp
    lower = ramp.numel() // 2
    return torch.tensor(ramp[:lower].tolist() + [0.0] * pad + ramp[lower:].tolist(), dtype=torch.float32)


def create_fp8_map(signed: bool = True, exponent_bits: int = 5, precision_bits: int = 2, total_bits: int = 8) -> Tensor:
    """Code book of a small floating-point format (sign / exponent / fraction), normalised to max 1
    and zero-padded to 256 entries: exponent field 0 holds the subnormals ``f * 2^-bias``, field
    ``E > 0`` holds ``(1 + f) * 2^-(E - bias - 1)`` with ``bias = 2^(exponent_bits - 1)`` -- the
    reference's convention, in which larger exponent fields mean SMALLER magnitudes (reference
    functional.py:227-293; pinned against a golden copy)."""
    if exponent_bits + precision_bits != total_bits - (1 if signed else 0):
        raise AssertionError("sign + exponent + precision bits must add up to total_bits")
    bias = 2 ** (exponent_bits - 1)
    fractions = [sum(((m >> (precision_bits - 1 - i)) & 1) * 2.0 ** -(i + 1) for i in range(precision_bits))
                 for m in range(2**precision_bits)]
    values: list[float] = []
    for field in range(2**exponent_bits):
        for f in fractions:
            v = f * 2.0**-bias if field == 0 else (1.0 + f) * 2.0 ** -(field - bias - 1)
            values.append(v)
            if signed:
                values.append(-v)
    if len(values) != 2**total_bits:
        raise AssertionError("fp8 map size mismatch")
    values += [0.0] * (256 - len(values))
    values.sort()
    code = torch.tensor(values, dtype=torch.float32)
    return code / code.max()


_4BIT_CODE_CACHE: dict = {}


def get_4bit_type(typename: str, device=None, blocksize: int = 64) -> Tensor:
    """16 fp32 code values, normalised to max |v| == 1 (reference functional.py:772-859).
    The device copy is built once per (type, device) and cloned afterwards: a host -> device transfer on every
    quantize_4bit call would put a synchronising copy on the hot path and break CUDA-graph capture."""
    if device is None:
        device = "cuda"
    key = (typename, str(torch.device(device)), blocksize)
    hit = _4BIT_CODE_CACHE.get(key)
    if hit is not None:
        return hit.clone()
    t = _build_4bit_type(typename, device, blocksize)
    _4BIT_CODE_CACHE[key] = t
    return t.clone()


def _build_4bit_type(typename: str, device, blocksize: int) -> Tensor:
    if typename == "nf4":
        data = list(_NF4_VALUES)
    elif typename == "fp4":
        data = list(_FP4_MAGNITUDES) + [(-m if m else 0.0) for m in _FP4_MAGNITUDES]  # table zero is +0.0
    elif typename == "int4":
        data = [7, 6, 5, 4, 3, 2, 1, 0, -0, -1, -2, -3, -4, -5, -6, -7]
    elif typename == "af4":
        if blocksize != 64:
            raise NotImplementedError("4-bit AbnormalFloats currently only support blocksize 64.")
        data = [-1.0, -0.69441008, -0.51243739, -0.3736951, -0.25607552, -0.14982478, -0.04934812, 0.0,
                0.04273164, 0.12934483, 0.21961274, 0.31675666, 0.42563882, 0.55496234, 0.72424863, 1.0][::-1]
    else:
        raise NotImplementedError(f"Typename {typename} not supported")
    t = torch.tensor(data, device=device)
    t.div_(t.abs().max())
    if t.numel() != 16:
        raise AssertionError("4-bit code must have 16 entries")
    return t


# ------------------------------------------------------------------------------------ QuantState
_DTYPE_NAMES = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16,
                "uint8": torch.uint8, "float64": torch.float64}


def _dtype_name(dt: torch.dtype) -> str:
    return str(dt).removeprefix("torch.")


class QuantState:
    """Everything needed to undo a blockwise quantisation (reference functional.py:420-610).

    ``absmax`` is fp32 per block -- or, with double quantisation, the uint8 codes of
    ``absmax - offset`` whose own state lives in ``state2`` (blocksize 256, dynamic map).
    The serialised form (``as_dict(packed=True)``) is the reference's: tensors under
    ``absmax / quant_map / nested_absmax / nested_quant_map`` plus one uint8 tensor
    ``quant_state.bitsandbytes__{nf4,fp4}`` holding the JSON of the scalar fields.
    """

    valid_quant_types = ("fp4", "nf4")
    valid_qs_type_keys = [f"bitsandbytes__{q}" for q in valid_quant_types]
    valid_qs_keys = ["absmax", "quant_map", "nested_absmax", "nested_quant_map", "quant_state", "quant_type",
                     "blocksize", "dtype", "shape", "nested_blocksize", "nested_dtype", "nested_offset"]

    def __init__(self, absmax, shape=None, code=None, blocksize=None, quant_type=None, dtype=None, offset=None,
                 state2=None):
        self.absmax = absmax
        self.shape = shape
        self.code = code
        self.dtype = dtype
        self.blocksize = blocksize
        self.quant_type = quant_type
        self.offset = offset
        self.state2 = state2
        self.nested = state2 is not None

    # FSDP resolves "quant_state.bitsandbytes__nf4" with getattr during state_dict traversal
    def __getattr__(self, name):
        if name.startswith("bitsandbytes__"):
            packed = self.as_dict(packed=True)
            key = "quant_state." + name
            if key in packed:
                return packed[key]
        raise AttributeError(f"'{type(self).__name__}' object has no attribute '{name}'")

    def __getitem__(self, idx):
        """Legacy list view: [absmax, shape, dtype, blocksize, [offset, state2] | None, quant_type]."""
        nested = [self.offset, self.state2] if self.nested else None
        return [self.absmax, self.shape, self.dtype, self.blocksize, nested, self.quant_type][idx]

    @classmethod
    def from_dict(cls, qs_dict: dict[str, Any], device) -> "QuantState":
        qs_dict = dict(qs_dict)
        packed_keys = [k for k, v in qs_dict.items() if "quant_state" in k and isinstance(v, Tensor)]
        if "quant_type" not in qs_dict:
            if not packed_keys:
                raise ValueError("Expected packed or unpacked quant_state items, found neither")
            if len(packed_keys) != 1 or packed_keys[0].split(".")[-1] not in cls.valid_qs_type_keys:
                raise ValueError(
                    f"There should be exactly one `quant_state` item with ending from {cls.valid_qs_type_keys}.\n"
                    f"Detected {packed_keys}.")
        if len(packed_keys) == 1:
            qs_dict.update(unpack_tensor_to_dict(qs_dict.pop(packed_keys[0])))
        flat = {k.split(".")[-1]: v for k, v in qs_dict.items()}
        unknown = set(flat) - set(cls.valid_qs_keys)
        if unknown:
            raise ValueError(f"unexpected quant_state keys: {sorted(unknown)}")

        offset = state2 = None
        if "nested_absmax" in flat:
            offset = torch.tensor(float(flat["nested_offset"])).to(device)
            state2 = cls(absmax=flat["nested_absmax"].to(device), blocksize=flat["nested_blocksize"],
                         code=flat["nested_quant_map"].to(device), dtype=_DTYPE_NAMES[flat["nested_dtype"]])
        shape = flat["shape"]
        return cls(quant_type=flat["quant_type"], absmax=flat["absmax"].to(device), blocksize=flat["blocksize"],
                   code=flat["quant_map"].to(device), dtype=_DTYPE_NAMES[flat["dtype"]],
                   shape=torch.Size(shape) if shape is not None else None, offset=offset, state2=state2)

    def as_dict(self, packed: bool = False) -> dict[str, Any]:
        d: dict[str, Any] = {
            "quant_type": self.quant_type,
            "absmax": self.absmax,
            "blocksize": self.blocksize,
            "quant_map": self.code,
            "dtype": _dtype_name(self.dtype),
            "shape": tuple(self.shape) if self.shape is not None else None,
        }
        if self.nested:
            d["nested_absmax"] = self.state2.absmax
            d["nested_blocksize"] = self.state2.blocksize
            d["nested_quant_map"] = self.state2.code.clone()  # safetensors drops shared tensors
            d["nested_dtype"] = _dtype_name(self.state2.dtype)
            d["nested_offset"] = self.offset.item()
        if not packed or self.quant_type is None:
            return d
        tensors = {k: v for k, v in d.items() if isinstance(v, Tensor)}
        scalars = {k: v for k, v in d.items() if not isinstance(v, Tensor)}
        tensors["quant_state.bitsandbytes__" + self.quant_type] = pack_dict_to_tensor(scalars)
        return tensors

    def to(self, device):
        self.code = self.code.to(device)
        self.absmax = self.absmax.to(device)
        if self.nested:
            self.offset = self.offset.to(device)
            self.state2.absmax = self.state2.absmax.to(device)
            self.state2.code = self.state2.code.to(device)

    def __eq__(self, other):
        if not isinstance(other, QuantState):
            return False

        def same_opt(a, b):
            if a is None or b is None:
                return a is b
            return bool(a == b)

        return (torch.allclose(self.absmax, other.absmax, atol=1e-6) and self.shape == other.shape
                and torch.allclose(self.code, other.code, atol=1e-6) and self.dtype == other.dtype
                and self.blocksize == other.blocksize and self.quant_type == other.quant_type
                and same_opt(self.offset, other.offset) and same_opt(self.state2, other.state2))

    __hash__ = None


# ------------------------------------------------------------------------------------ 8-bit blockwise
def _dynamic_code(device) -> Tensor:
    if "dynamic" not in name2qmap:
        name2qmap["dynamic"] = create_dynamic_map()
    name2qmap["dynamic"] = name2qmap["dynamic"].to(device)
    return name2qmap["dynamic"]


def quantize_blockwise(A: Tensor, code: Optional[Tensor] = None, absmax: Optional[Tensor] = None,
                       out: Optional[Tensor] = None, blocksize: int = 4096, nested: bool = False):
    """8-bit blockwise quantisation with the (default: dynamic) 256-entry code book.
    Returns ``(codes uint8 like A, QuantState)``."""
    if code is None:
        code = _dynamic_code(A.device)
    q, _absmax = _ops_ns.quantize_blockwise.default(A, code.to(A.device), blocksize)
    if nested:
        offset = _absmax.mean()
        qabsmax, state2 = quantize_blockwise(_absmax - offset, blocksize=blocksize, nested=False)
        state = QuantState(absmax=qabsmax, code=code.to(A.device, copy=True), blocksize=blocksize, dtype=A.dtype,
                           offset=offset, state2=state2)
    else:
        state = QuantState(absmax=_absmax, code=code.to(A.device, copy=True), blocksize=blocksize, dtype=A.dtype)
    if out is not None:
        out.copy_(q)
        q = out
    if absmax is not None:
        absmax.copy_(state.absmax)
        state.absmax = absmax
    return q, state


def dequantize_blockwise(A: Tensor, quant_state: Optional[QuantState] = None, absmax: Optional[Tensor] = None,
                         code: Optional[Tensor] = None, out: Optional[Tensor] = None, blocksize: int = 4096,
                         nested: bool = False) -> Tensor:
    if quant_state is None and absmax is None:
        raise ValueError("either quant_state or absmax must be given")
    if quant_state is None:
        if code is None:
            code = _dynamic_code(A.device)
        quant_state = QuantState(absmax=absmax, code=code, blocksize=blocksize, dtype=torch.float32)
    absmax = quant_state.absmax
    if quant_state.nested:
        absmax = dequantize_blockwise(quant_state.absmax, quant_state.state2) + quant_state.offset
        if absmax.dtype != torch.float32:
            absmax = absmax.float()
    if out is not None:
        _ops_ns.dequantize_blockwise.out(A, absmax, quant_state.code.to(A.device), quant_state.blocksize,
                                         quant_state.dtype, out=out)
        return out
    return _ops_ns.dequantize_blockwise.default(A, absmax, quant_state.code.to(A.device), quant_state.blocksize,
                                                quant_state.dtype)


# ------------------------------------------------------------------------------------ 4-bit blockwise
def quantize_4bit(A: Tensor, absmax: Optional[Tensor] = None, out: Optional[Tensor] = None, blocksize: Optional[int] = None,
                  compress_statistics: bool = False, quant_type: str = "fp4", quant_storage=torch.uint8):
    """Blockwise 4-bit (NF4 / FP4) quantisation; two codes per byte, element 2b in the high
    nibble.  ``compress_statistics`` quantises ``absmax - mean`` to 8 bits (blocksize 256)."""
    if blocksize is None:
        blocksize = 64
    input_shape = A.shape
    _out, _absmax = _ops_ns.quantize_4bit.default(A, blocksize, quant_type, quant_storage)
    code = get_4bit_type(quant_type, device=A.device)
    if compress_statistics:
        offset = _absmax.mean()
        qabsmax, state2 = quantize_blockwise(_absmax - offset, blocksize=256)
        del _absmax
        state = QuantState(absmax=qabsmax, shape=input_shape, dtype=A.dtype, blocksize=blocksize, code=code,
                           quant_type=quant_type, offset=offset, state2=state2)
    else:
        state = QuantState(absmax=_absmax, shape=input_shape, dtype=A.dtype, blocksize=blocksize, code=code,
                           quant_type=quant_type)
    if out is not None:
        out.copy_(_out)
        _out = out
    if absmax is not None:
        absmax.copy_(state.absmax)
        state.absmax = absmax
    return _out, state


def quantize_fp4(A, absmax=None, out=None, blocksize=None, compress_statistics=False, quant_storage=torch.uint8):
    return quantize_4bit(A, absmax, out, blocksize, compress_statistics, "fp4", quant_storage)


def quantize_nf4(A, absmax=None, out=None, blocksize=None, compress_statistics=False, quant_storage=torch.uint8):
    return quantize_4bit(A, absmax, out, blocksize, compress_statistics, "nf4", quant_storage)


def dequantize_4bit(A: Tensor, quant_state: Optional[QuantState] = None, absmax: Optional[Tensor] = None,
                    out: Optional[Tensor] = None, blocksize: Optional[int] = None, quant_type: str = "fp4") -> Tensor:
    if blocksize is None:
        blocksize = 64
    if quant_state is None:
        if absmax is None or out is None:
            raise ValueError("without a quant_state, both absmax and out must be given")
        quant_state = QuantState(absmax=absmax, shape=out.shape, dtype=out.dtype, blocksize=blocksize,
                                 quant_type=quant_type)
    else:
        absmax = quant_state.absmax
    if quant_state.nested:
        absmax = dequantize_blockwise(quant_state.absmax, quant_state.state2) + quant_state.offset
        if absmax.dtype != torch.float32:
            absmax = absmax.float()
    if out is not None:
        _ops_ns.dequantize_4bit.out(A, absmax, quant_state.blocksize, quant_state.quant_type, quant_state.shape,
                                    quant_state.dtype, out=out)
    else:
        out = _ops_ns.dequantize_4bit.default(A, absmax, quant_state.blocksize, quant_state.quant_type,
                                              quant_state.shape, quant_state.dtype)
    if A.shape[0] == 1:  # a transposed [1, n] packed weight: hand back the matching orientation
        return out.t()
    return out


def dequantize_fp4(A, quant_state=None, absmax=None, out=None, blocksize=None):
    return dequantize_4bit(A, quant_state, absmax, out, blocksize, "fp4")


def dequantize_nf4(A, quant_state=None, absmax=None, out=None, blocksize=None):
    return dequantize_4bit(A, quant_state, absmax, out, blocksize, "nf4")


def gemv_4bit(A: Tensor, B: Tensor, out: Optional[Tensor] = None, transposed_A=False, transposed_B=False, state=None):
    """Legacy single-token 4-bit mat-vec (reference functional.py:1300-1334)."""
    if state is None:
        raise ValueError("state cannot be None. gemv_4bit() requires the state from quantize_4bit()")
    absmax = state.absmax
    if state.nested:
        absmax = dequantize_blockwise(absmax, state.state2) + state.offset
    if out is not None:
        _ops_ns.gemv_4bit.out(A, B, state.shape, absmax, state.code, state.blocksize, out=out)
        return out
    return _ops_ns.gemv_4bit.default(A, B, state.shape, absmax, state.code, state.blocksize)


# ------------------------------------------------------------------------------------ LLM.int8()
def int8_linear_matmul(A: Tensor, B: Tensor, out: Optional[Tensor] = None, dtype=torch.int32):
    """int32 = A[..., K] (int8) . B[N, K]^T (int8), exact."""
    if out is not None:
        _ops_ns.int8_linear_matmul.out(A, B, out)
        return out
    return _ops_ns.int8_linear_matmul.default(A, B)


def int8_mm_dequant(A: Tensor, row_stats: Tensor, col_stats: Tensor, out: Optional[Tensor] = None,
                    bias: Optional[Tensor] = None):
    result = _ops_ns.int8_mm_dequant.default(A, row_stats, col_stats, dtype=torch.float16, bias=bias)
    if out is not None:
        return out.copy_(result)
    return result


def int8_double_quant(A: Tensor, col_stats=None, row_stats=None, out_col=None, out_row=None, threshold: float = 0.0):
    if any(x is not None for x in (col_stats, row_stats, out_col, out_row)):
        raise ValueError("preallocated outputs are not supported")
    return _ops_ns.int8_double_quant.default(A, threshold=threshold)


def int8_vectorwise_dequant(A: Tensor, stats: Tensor) -> Tensor:
    return _ops_ns.int8_vectorwise_dequant.default(A, stats)


def int8_vectorwise_quant(A: Tensor, threshold: float = 0.0):
    """Row-wise absmax int8 quantisation; with ``threshold > 0`` also returns the indices of
    the columns holding any |a| >= threshold (those entries are written as 0)."""
    return _ops_ns.int8_vectorwise_quant.default(A, threshold)


# ------------------------------------------------------------------------------------ small compat helpers
def get_ptr(A: Optional[Tensor]) -> Optional[ct.c_void_p]:
    return None if A is None else ct.c_void_p(A.data_ptr())


def is_on_gpu(tensors) -> bool:
    on = [t for t in tensors if t is not None]
    devices = {(t.device.type, t.device.index) for t in on}
    if any(d[0] != "cuda" for d in devices):
        raise RuntimeError("All input tensors need to be on a CUDA device: " + str([(t.shape, t.device) for t in on]))
    if len(devices) > 1:
        raise RuntimeError("Input tensors need to be on the same GPU: " + str([(t.shape, t.device) for t in on]))
    return True


# ------------------------------------------------------------------------------------ optimizers (SURVEY.md 8 f-4)
def is_on_gpu_or_paged(tensors) -> bool:
    """Like is_on_gpu, but a managed ("paged") tensor -- a CPU tensor over cudaMallocManaged memory -- is accepted."""
    on = [t for t in tensors if t is not None and not getattr(t, "is_paged", False)]
    return is_on_gpu(on)


def optimizer_update_32bit(optimizer_name: str, g: Tensor, p: Tensor, state1: Tensor, beta1: float, eps: float, step: int,
                           lr: float, state2: Optional[Tensor] = None, beta2: float = 0.0, beta3: float = 0.0,
                           alpha: float = 0.0, weight_decay: float = 0.0, gnorm_scale: float = 1.0,
                           unorm_vec: Optional[Tensor] = None, max_unorm: float = 0.0, skip_zeros=False) -> None:
    """In-place optimizer step with fp32 state and fp32 / fp16 / bf16 gradients and parameters (reference
    functional.py:1080-1166).  optimizer_name: adam, momentum, rmsprop, adagrad, lion, ademamix, lamb, lars."""
    param_norm = 0.0
    if max_unorm > 0.0:
        param_norm = float(torch.norm(p.data.float()))
    is_on_gpu_or_paged([g, p, state1, state2, unorm_vec])
    _ops_ns.optimizer_update_32bit(optimizer_name, g, p, state1, state2, unorm_vec, max_unorm, param_norm, beta1, beta2,
                                   beta3, alpha, eps, weight_decay, step, lr, gnorm_scale, skip_zeros)


def optimizer_update_8bit_blockwise(optimizer_name: str, g: Tensor, p: Tensor, state1: Tensor, state2: Optional[Tensor],
                                    beta1: float, beta2: float, beta3: float, alpha: float, eps: float, step: int,
                                    lr: float, qmap1: Tensor, qmap2: Optional[Tensor], absmax1: Tensor,
                                    absmax2: Optional[Tensor], weight_decay: float = 0.0, gnorm_scale: float = 1.0,
                                    skip_zeros=False) -> None:
    """In-place optimizer step with blockwise (256) 8-bit state (reference functional.py:1169-1213)."""
    is_on_gpu_or_paged([p, g, state1, state2, qmap1, qmap2, absmax1, absmax2])
    _ops_ns.optimizer_update_8bit_blockwise(optimizer_name, g, p, state1, state2, beta1, beta2, beta3, alpha, eps, step, lr,
                                            qmap1, qmap2, absmax1, absmax2, weight_decay, gnorm_scale, skip_zeros)


def optimizer_update_32bit_multi(optimizer_name: str, g: Sequence[Tensor], p: Sequence[Tensor], state1: Sequence[Tensor],
                                 beta1: float, eps: float, step: Sequence[Union[int, Tensor]], lr: Union[float, Tensor],
                                 state2: Optional[Sequence[Tensor]] = None, beta2: float = 0.0, beta3: float = 0.0,
                                 alpha: float = 0.0, weight_decay: float = 0.0, gnorm_scale: float = 1.0,
                                 skip_zeros=False) -> None:
    """``optimizer_update_32bit`` for several parameters at once: one kernel launch per
    ``backends.cuda.optimizer_multi_capacity()`` parameters instead of one per parameter, with the same results bit
    for bit.  g, p, state1, step (and state2 for adam / ademamix) list one entry per parameter; every other argument is
    shared.  All tensors on one GPU (paged state allowed); no trust ratio (max_unorm: LAMB / LARS take the
    single-tensor call).

    Capturable form: when ``step`` lists one-element int32 CUDA tensors, one per parameter, the call advances each by
    one on the GPU and updates with the advanced steps, and ``lr`` may be a one-element float32 CUDA tensor.  The call
    then reads nothing on the host, so a CUDA graph that captured it uses the current steps and ``lr`` at every replay.
    The results are those of the integer form given the same steps and ``lr``, bit for bit."""
    _cuda_backend.optimizer_update_32bit_multi(optimizer_name, g, p, state1, state2, beta1, beta2, beta3, alpha, eps,
                                               weight_decay, step, lr, gnorm_scale, skip_zeros)


def optimizer_update_8bit_blockwise_multi(optimizer_name: str, g: Sequence[Tensor], p: Sequence[Tensor],
                                          state1: Sequence[Tensor], state2: Optional[Sequence[Tensor]], beta1: float,
                                          beta2: float, beta3: float, alpha: float, eps: float,
                                          step: Sequence[Union[int, Tensor]], lr: Union[float, Tensor], qmap1: Tensor, qmap2: Optional[Tensor], absmax1: Sequence[Tensor],
                                          absmax2: Optional[Sequence[Tensor]], weight_decay: float = 0.0,
                                          gnorm_scale: float = 1.0, skip_zeros=False) -> None:
    """``optimizer_update_8bit_blockwise`` for several parameters at once: one kernel launch per
    ``backends.cuda.optimizer_multi_capacity()`` parameters instead of one per parameter, with the same results bit
    for bit.  g, p, state1, absmax1, step (and state2 / absmax2 for adam / ademamix) list one entry per parameter; the
    code books and every other argument are shared.  Device steps and ``lr``: as ``optimizer_update_32bit_multi``."""
    _cuda_backend.optimizer_update_8bit_blockwise_multi(optimizer_name, g, p, state1, state2, beta1, beta2, beta3, alpha,
                                                        eps, step, lr, qmap1, qmap2, absmax1, absmax2, weight_decay,
                                                        gnorm_scale, skip_zeros)


class GlobalPageManager:
    """Registry of the managed ("paged") optimizer-state tensors (reference functional.py:25-48)."""

    _instance = None

    def __init__(self):
        raise RuntimeError("Call get_instance() instead")

    def initialize(self):
        self.paged_tensors = []

    @classmethod
    def get_instance(cls):
        if cls._instance is None:
            cls._instance = cls.__new__(cls)
            cls._instance.initialize()
        return cls._instance

    def prefetch_all(self, to_cpu=False):
        for t in self.paged_tensors[::-1]:  # the first ones are used first: bring them in last
            prefetch_tensor(t, to_cpu)


def get_paged(*shape, dtype=torch.float32, device=None):
    """A tensor over cudaMallocManaged memory: addressable from the host and from every GPU, migrated on demand
    (reference functional.py:91-100).  It is a CPU tensor to PyTorch; the kernels receive its raw pointer."""
    import numpy as np

    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    count = 1
    for d in shape:
        count *= int(d)
    num_bytes = dtype.itemsize * count
    ptr = lib.cget_managed_ptr(num_bytes)
    lib.check("get_paged")
    if not ptr:
        raise RuntimeError(f"get_paged: could not allocate {num_bytes} bytes of managed memory")
    buf = (ct.c_uint8 * num_bytes).from_address(ptr)
    out = torch.frombuffer(np.ctypeslib.as_array(buf), dtype=dtype, count=count).view(shape)
    out.is_paged = True
    out.page_deviceid = device.index
    return out


def prefetch_tensor(A: Tensor, to_cpu=False):
    assert getattr(A, "is_paged", False), "Only paged tensors can be prefetched!"
    lib.cprefetch(A.data_ptr(), A.nbytes, -1 if to_cpu else A.page_deviceid)
    lib.check("prefetch_tensor")


def fill(A: Tensor, value, device=None, prefetch=True):
    """A[:] = value through the native element-wise helper (works on managed tensors; reference functional.py:142)."""
    if A.dtype == torch.float32:
        lib.cfill_fp32(A.data_ptr(), None, float(value), A.numel())
    elif A.dtype == torch.uint8:
        lib.cfill_uint8(A.data_ptr(), None, int(value), A.numel())
    else:
        raise NotImplementedError(f"fill: dtype {A.dtype}")
    lib.check("fill")
    if getattr(A, "is_paged", False):
        torch.cuda.synchronize()


def has_avx512bf16() -> bool:  # probed by the reference's Linear4bit; never true here (no CPU path)
    return False


class CUBLAS_Context:
    """Kept for API compatibility: the int8 GEMM is our own kernel, the "context" an opaque token."""

    _instance = None

    def __init__(self):
        raise RuntimeError("Call get_instance() instead")

    @classmethod
    def get_instance(cls):
        if cls._instance is None:
            cls._instance = cls.__new__(cls)
            cls._instance.context = {}
        return cls._instance

    def get_context(self, device):
        if device.index not in self.context:
            self.context[device.index] = ct.c_void_p(lib.get_context())
        return self.context[device.index]


def _enumerate_kbit_values(total_bits: int):  # helper for tests that build small code books
    return list(itertools.product([0, 1], repeat=total_bits))
