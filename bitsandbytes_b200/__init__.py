"""bitsandbytes_b200 -- an H100-native (sm_90a) implementation of the bitsandbytes
quantized-linear hot path: NF4/FP4 4-bit dequant-fused GEMM, LLM.int8() and blockwise
quantize/dequantize, behind the ``bnb.functional`` / ``bnb.nn`` API surface.

Layout (only what the path needs):
    cextension.py      loads libbitsandbytes_b200.so (C ABI declared in include/bitsandbytes_b200.h)
    csrc/              CUDA kernels + the extern "C" boundary
    _ops.py            torch.library schemas (namespace ``bitsandbytes::``) + the CUDA kernels' host side
    functional.py      QuantState, quantize/dequantize_{blockwise,4bit}, int8_* ...
    autograd/          matmul_4bit / matmul (MatMul4Bit, MatMul8bitLt)
    nn/                Linear4bit, Params4bit, Linear8bitLt, Int8Params
    parallel.py        column-sharded Linear4bit over NCCL (one process per GPU)
    optim/             optimizers with 32-bit / blockwise 8-bit state (Adam, AdamW, Lion, SGD, RMSprop, ...)
"""
__version__ = "0.1.0"

from . import cextension  # noqa: F401  (loads the native library; raises on first use if missing)

_LAZY = ("functional", "nn", "autograd", "utils", "parallel", "_ops", "optim")


def __getattr__(name):
    import importlib

    if name in _LAZY:
        return importlib.import_module(f"{__name__}.{name}")
    if name in ("matmul", "matmul_4bit", "MatmulLtState"):
        mod = importlib.import_module(f"{__name__}.autograd._functions")
        return getattr(mod, name)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")


# probed by HF Transformers' bitsandbytes integration (reference __init__.py:25-33)
features = {"multi_backend"}
supported_torch_devices = {"cuda"}
