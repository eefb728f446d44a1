"""GPU parity against the committed golden fixtures (tests/golden/reference_vectors_*.npz: outputs of the
reference's own CPU backend and pure-torch kernels on seeded inputs, edge sizes included), through the
product's C ABI.  The checker (tests/_golden_check.py) is validated on CPU with the oracle as the
implementation (tests/test_oracle_pinned.py).  This file sorts last on purpose: it was added after the
round's last GPU run, so a surprise here cannot hide the results of the suites above."""
import numpy as np
import pytest
import torch

from tests import _native as nat

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------- golden vectors
# The reference-generated fixtures (tests/golden/reference_vectors_*.npz: the reference's own CPU
# backend and pure-torch kernels on seeded inputs, edge sizes included) through the product's C ABI.
def _gpu_quantize(A, dtype, bs, qt, code):
    if dtype == "fp32":
        t = torch.from_numpy(np.ascontiguousarray(A, dtype=np.float32).reshape(-1).copy())
    else:
        t = torch.from_numpy(np.ascontiguousarray(A).reshape(-1).view(np.int16).copy()).view(nat.DTYPE[dtype])
    c = torch.from_numpy(code.copy()).cuda() if code is not None else None
    out, absmax = nat.quantize(nat.lib, t.cuda(), bs, qt, c, dtype)
    nat.check()
    return out.cpu().numpy(), absmax.cpu().numpy()


def _gpu_dequantize(codes, absmax, bs, n, qt, code, out_dtype):
    c = torch.from_numpy(code.copy()).cuda() if code is not None else None
    d = nat.dequantize(nat.lib, torch.from_numpy(np.ascontiguousarray(codes).copy()).cuda(),
                       torch.from_numpy(np.ascontiguousarray(absmax).copy()).cuda(), bs, n, qt, c, out_dtype)
    nat.check()
    d = d.cpu()
    return d.numpy() if out_dtype == "fp32" else d.view(torch.int16).numpy().view(np.uint16)


@pytest.mark.parametrize("name", ["a", "b", "c", "d", "e", "f", "g", "h"])
def test_golden_vectors_8bit(name):
    from tests import _golden_check as gc

    gc.check_8bit(gc.load(), name, _gpu_quantize, _gpu_dequantize)


@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("name", ["a", "b", "c", "d", "e", "f", "g", "h", "i"])
def test_golden_vectors_4bit(qt, name):
    from tests import _golden_check as gc

    gc.check_4bit(gc.load(), qt, name, _gpu_quantize, _gpu_dequantize)


# ---------------------------------------------------------------------------- golden vectors
def _gpu_gemm4(x_bits, dt, packed, absmax, a8, code2, offset, bias_bits, M, N, K, bs, qt):
    x = nat.from_bits(x_bits, dt).reshape(M, K)
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a).copy()).cuda()  # noqa: E731
    off = None if offset is None else torch.tensor([offset], dtype=torch.float32, device="cuda")
    bias = None if bias_bits is None else nat.from_bits(bias_bits, dt)
    out = nat.gemm_4bit(nat.lib, x, t(packed), t(absmax), M, N, K, bs, qt, dt, bias, t(a8), t(code2), off)
    nat.check()
    return out.double().cpu().numpy()


@pytest.mark.parametrize("path", [-1, 1], ids=["auto", "tcgen05"])
@pytest.mark.parametrize("name", ["plain", "nested", "fp16"])
def test_golden_vectors_gemm4(name, path):
    """The reference's public API on its CPU backend (tests/golden/reference_vectors_*.npz) vs the product kernels
    (the decode kernel by default at these M; the wgmma kernel when forced)."""
    from tests import _golden_check as gc

    nat.lib.cbnb_b200_gemm_4bit_force_path(path)
    try:
        gc.check_gemm4(gc.load(), name, _gpu_gemm4)
    finally:
        nat.lib.cbnb_b200_gemm_4bit_force_path(-1)


# ---------------------------------------------------------------------------- golden vectors
def test_golden_vectors_int8_gemm_and_dequant():
    """tests/golden/reference_vectors_*.npz (the reference's int8_linear_matmul / int8_mm_dequant on CPU) through the
    C ABI: the int8 GEMM exactly, the dequantisation within one fp16 ulp (the reference's torch kernel multiplies
    in a different order)."""
    from tests import _golden_check as gc

    def gemm(A, B):
        M, K = A.shape
        N = B.shape[0]
        a, b = torch.from_numpy(A.copy()).cuda(), torch.from_numpy(B.copy()).cuda()
        C = torch.full((M, N), -7, device="cuda", dtype=torch.int32)
        rc = nat.lib.cigemmlt_32(nat.lib.get_context(), N, M, K, b.data_ptr(), a.data_ptr(), C.data_ptr(), None, K, K, N,
                                 nat.stream())
        torch.cuda.synchronize()
        nat.check()
        assert rc == 0
        return C.cpu().numpy()

    def dequant(C, rs, cs, bias_bits):
        rows, cols = C.shape
        c = torch.from_numpy(C.copy()).cuda()
        r, s = torch.from_numpy(rs.copy()).cuda(), torch.from_numpy(cs.copy()).cuda()
        bias = None if bias_bits is None else nat.from_bits(bias_bits, "fp16")
        out = torch.zeros((rows, cols), device="cuda", dtype=torch.float16)
        nat.lib.cdequant_mm_int32_fp16(c.data_ptr(), r.data_ptr(), s.data_ptr(), out.data_ptr(), nat.ptr(bias), rows, cols,
                                       nat.stream())
        torch.cuda.synchronize()
        nat.check()
        return nat.to_bits(out)

    gc.check_int8_gemm(gc.load(), gemm, dequant)
