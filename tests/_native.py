"""Test-side helpers: raw C-ABI calls on torch-owned device buffers, for both our library
and (when present) the reference CUDA library built by oracle/Makefile."""
import ctypes as ct

import numpy as np
import torch

import oracle
from bitsandbytes_b200 import cextension

lib = cextension.lib
DTYPE = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
DTYPE_ID = {"fp32": 0, "fp16": 1, "bf16": 2}
QT_ID = {None: 0, "fp4": 1, "nf4": 2}

_ref = None


def ref_cuda():
    """The reference CUDA library (same C ABI, built by oracle/Makefile from the reference sources): the STRICT
    oracle of the GPU tests.  Not built -> the calling test is skipped, visibly, in the pytest summary; built but
    not loadable -> the calling test FAILS (a silent downgrade to the looser CPU-oracle bounds is not allowed)."""
    import pytest

    global _ref
    if _ref is None:
        path = oracle.ref_cuda_library_path()
        if path is None or not path.exists():
            _ref = False
        else:
            try:
                dll = ct.CDLL(str(path))
            except OSError as e:
                pytest.fail(f"the reference CUDA library exists at {path} but does not load: {e}")
            for name, (argtypes, restype) in cextension._signatures().items():
                if name.startswith("cbnb_b200"):
                    continue
                fn = getattr(dll, name, None)
                if fn is not None:
                    fn.argtypes = argtypes
                    fn.restype = restype
            _ref = dll
    if _ref is False:
        pytest.skip("reference CUDA library not built (oracle/_ref/libbitsandbytes_cuda_ref.so): strict parity not checked")
    return _ref


def stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()


def to_bits(t: torch.Tensor) -> np.ndarray:
    t = t.detach().contiguous().cpu()
    if t.dtype in (torch.bfloat16, torch.float16):
        return t.view(torch.int16).numpy().view(np.uint16)
    return t.numpy()


def from_bits(a: np.ndarray, dtype: str, device="cuda") -> torch.Tensor:
    if dtype == "fp32":
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).view(DTYPE[dtype]).to(device)


def quantize(L, A: torch.Tensor, blocksize: int, qt, code=None, dtype="fp32"):
    """reference-ABI quantize (legacy default stream) on library L."""
    n = A.numel()
    nblocks = -(n // -blocksize)
    absmax = torch.full((nblocks,), float("nan"), device="cuda", dtype=torch.float32)
    out = torch.zeros(n if qt is None else (n + 1) // 2, device="cuda", dtype=torch.uint8)
    suffix = "" if qt is None else f"_{qt}"
    fn = getattr(L, f"cquantize_blockwise_{dtype}{suffix}")
    torch.cuda.synchronize()
    fn(ptr(code), ptr(A), ptr(absmax), ptr(out), blocksize, n)
    torch.cuda.synchronize()
    return out, absmax


def dequantize(L, codes: torch.Tensor, absmax: torch.Tensor, blocksize: int, n: int, qt, code=None, dtype="fp32"):
    out = torch.full((n,), float("nan"), device="cuda", dtype=DTYPE[dtype])  # an element never written fails
    suffix = "" if qt is None else f"_{qt}"
    fn = getattr(L, f"cdequantize_blockwise_{dtype}{suffix}")
    fn(ptr(code), ptr(codes), ptr(absmax), ptr(out), blocksize, n, stream())
    torch.cuda.synchronize()
    return out


def gemm_4bit(L, x, packed, absmax, M, N, K, blocksize, qt, dtype, bias=None, absmax_8bit=None, absmax_code=None,
              absmax_offset=None):
    out = torch.full((M, N), float("nan"), device="cuda", dtype=DTYPE[dtype])
    fn = getattr(L, f"cgemm_4bit_{dtype}")
    fn(ptr(x), ptr(packed), ptr(absmax), ptr(absmax_8bit), ptr(absmax_code), ptr(absmax_offset), ptr(out), ptr(bias),
       M, N, K, blocksize, QT_ID[qt], stream())
    torch.cuda.synchronize()
    return out


def check():
    lib.check("test call")
