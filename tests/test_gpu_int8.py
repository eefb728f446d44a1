"""GPU parity: LLM.int8() pieces through the C ABI.

Bars: int8 GEMM exact (integers); row statistics exact; int8 codes bit-equal to the
reference CUDA kernel (and within +-1 of the CPU oracle only where a*127/absmax sits on a
rounding boundary, the reference's own tolerance, reference tests/test_functional.py:508-536);
dequant epilogue bit-equal to the reference kernel's formula.
"""
import numpy as np
import pytest
import torch

import oracle
from tests import _native as nat

pytestmark = pytest.mark.gpu


def _acts(rows, cols, dtype=torch.float16, outliers=5, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + rows * 3 + cols)
    A = torch.randn(rows, cols, generator=g)
    if outliers:
        idx = torch.randperm(cols, generator=g)[:outliers]
        A[:, idx] = 8.0  # reference benchmarking/matmul_benchmark.py:47-48
        A[rows // 2, (idx[0] + 1) % cols] = -6.5
    return A.to(dtype).cuda()


@pytest.mark.parametrize("rows,cols", [(7, 96), (64, 4096), (33, 1000), (5, 8200), (128, 11008), (1, 64)])
@pytest.mark.parametrize("threshold", [0.0, 6.0])
def test_vector_quant_vs_reference_and_oracle(rows, cols, threshold):
    A = _acts(rows, cols)
    q = torch.zeros(rows, cols, device="cuda", dtype=torch.int8)
    stats = torch.zeros(rows, device="cuda")
    nat.lib.cint8_vector_quant(A.data_ptr(), q.data_ptr(), stats.data_ptr(), threshold, rows, cols, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    oq, ostats = oracle.int8_vector_quant(nat.to_bits(A), threshold)
    np.testing.assert_array_equal(stats.cpu().numpy(), ostats)
    d = np.abs(q.cpu().numpy().astype(int) - oq.astype(int))
    assert d.max() <= 1 and (d != 0).mean() < 1e-3
    ref = nat.ref_cuda()
    if ref is not None:
        rq = torch.zeros_like(q)
        rstats = torch.zeros_like(stats)
        ref.cint8_vector_quant(A.data_ptr(), rq.data_ptr(), rstats.data_ptr(), threshold, rows, cols, nat.stream())
        torch.cuda.synchronize()
        assert torch.equal(rstats, stats)
        assert torch.equal(rq, q), f"{(rq != q).sum().item()} int8 codes differ from the reference CUDA kernel"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_vector_quant_outlier_flags(dtype):
    rows, cols = 48, 4096
    A = _acts(rows, cols, dtype, outliers=7)
    q = torch.zeros(rows, cols, device="cuda", dtype=torch.int8)
    stats = torch.zeros(rows, device="cuda")
    flags = torch.zeros(cols, device="cuda", dtype=torch.int32)
    nat.lib.cbnb_b200_int8_vector_quant_flags(A.data_ptr(), q.data_ptr(), stats.data_ptr(), flags.data_ptr(), 6.0, rows,
                                              cols, 1 if dtype == torch.float16 else 2, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    want = (A.float().abs() >= 6.0).any(dim=0)
    assert torch.equal(flags.bool(), want)
    masked = torch.where(A.float().abs() < 6.0, A.float().abs(), torch.zeros((), device="cuda"))
    assert torch.equal(stats, masked.amax(dim=1))
    assert (q[(A.float().abs() >= 6.0)] == 0).all()


@pytest.mark.parametrize("M,N,K", [(9, 24, 64), (128, 256, 128), (130, 300, 192), (1, 64, 4096), (300, 1000, 1024),
                                   (4096, 512, 4096), (77, 11008, 256), (5, 40, 16), (130, 129, 48)])
def test_int8_gemm_exact(M, N, K):
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    A = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8).cuda()
    B = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8).cuda()
    C = torch.full((M, N), -7, device="cuda", dtype=torch.int32)
    rc = nat.lib.cigemmlt_32(nat.lib.get_context(), N, M, K, B.data_ptr(), A.data_ptr(), C.data_ptr(), None, K, K, N,
                             nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    if M * N * K <= 2**24:
        np.testing.assert_array_equal(C.cpu().numpy(), oracle.int8_gemm(A.cpu().numpy(), B.cpu().numpy()))
    want = (A.double() @ B.double().t()).to(torch.int32)  # exact: |sum| < 2^53
    assert torch.equal(C, want)
    ref = nat.ref_cuda()
    if ref is not None and K % 4 == 0:
        ctx = ref.get_context()
        R = torch.zeros_like(C)
        rc = ref.cigemmlt_32(ctx, N, M, K, B.data_ptr(), A.data_ptr(), R.data_ptr(), None, K, K, N, nat.stream())
        torch.cuda.synchronize()
        if rc == 0:
            assert torch.equal(R, C)


def test_int8_gemm_rejects_unaligned_k():
    A = torch.zeros(4, 20, dtype=torch.int8, device="cuda")
    B = torch.zeros(8, 20, dtype=torch.int8, device="cuda")
    C = torch.zeros(4, 8, dtype=torch.int32, device="cuda")
    rc = nat.lib.cigemmlt_32(nat.lib.get_context(), 8, 4, 20, B.data_ptr(), A.data_ptr(), C.data_ptr(), None, 20, 20, 8,
                             nat.stream())
    assert rc == 100  # caller falls back, as for the reference's K % 4 != 0 case


@pytest.mark.parametrize("rows,cols", [(9, 24), (64, 4096), (33, 1001), (4096, 512), (70000, 12)])
@pytest.mark.parametrize("with_bias", [False, True])
def test_mm_dequant_kernel(rows, cols, with_bias):
    g = torch.Generator(device="cpu").manual_seed(rows + cols)
    C = torch.randint(-2**20, 2**20, (rows, cols), generator=g, dtype=torch.int32).cuda()
    rs = (torch.rand(rows, generator=g) * 3 + 0.1).cuda()
    cs = (torch.rand(cols, generator=g) * 2 + 0.1).cuda()
    bias = torch.randn(cols, generator=g).half().cuda() if with_bias else None
    out = torch.zeros(rows, cols, device="cuda", dtype=torch.float16)
    nat.lib.cdequant_mm_int32_fp16(C.data_ptr(), rs.data_ptr(), cs.data_ptr(), out.data_ptr(), nat.ptr(bias), rows, cols,
                                   nat.stream())
    torch.cuda.synchronize()
    nat.check()
    want = oracle.int8_mm_dequant(C.cpu().numpy(), rs.cpu().numpy(), cs.cpu().numpy(),
                                  nat.to_bits(bias) if bias is not None else None)
    np.testing.assert_array_equal(nat.to_bits(out), want)
    ref = nat.ref_cuda()
    if ref is not None:
        r = torch.zeros_like(out)
        ref.cdequant_mm_int32_fp16(C.data_ptr(), rs.data_ptr(), cs.data_ptr(), r.data_ptr(), nat.ptr(bias), rows, cols,
                                   nat.stream())
        torch.cuda.synchronize()
        assert torch.equal(r.view(torch.int16), out.view(torch.int16))


def expected_scaled_mm(C: torch.Tensor, SCA: torch.Tensor, SCB: torch.Tensor, bias, dtype) -> torch.Tensor:
    """int8_scaled_mm's output from its exact int32 accumulators, by the pinned C restatement of the dequant formula.
    fp16: fp16(fma(C*SCA*SCB, 1/127^2, bias)).  bf16: the fp16 result without bias, the bias added in fp32 and rounded
    to fp16, then rounded to bf16 -- the order of the reference's unfused chain, which the fused epilogue keeps."""
    C, SCA, SCB = C.cpu().numpy(), SCA.cpu().numpy(), SCB.cpu().numpy()
    if dtype == torch.float16:
        return nat.from_bits(oracle.int8_mm_dequant(C, SCA, SCB, nat.to_bits(bias) if bias is not None else None), "fp16")
    h = oracle.widen(oracle.int8_mm_dequant(C, SCA, SCB), "fp16")
    if bias is not None:
        h = oracle.widen(oracle.round_to(h + oracle.widen(nat.to_bits(bias), "bf16"), "fp16"), "fp16")
    return nat.from_bits(oracle.round_to(h, "bf16"), "bf16")


# K = 16 / 80 / 208: a k-block of 128 bytes that is mostly past the end of K; N < 8 and N = 129: one partial column
# pair, and a second tile with one column; M = 1: one valid row in a 128-row tile
@pytest.mark.parametrize("M,N,K", [(9, 24, 64), (200, 384, 256), (4096, 1024, 512), (33, 5, 16), (1, 129, 80),
                                   (130, 129, 208), (1, 7, 208)])
@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_fused_scaled_mm_equals_gemm_then_dequant(M, N, K, with_bias, dtype):
    g = torch.Generator(device="cpu").manual_seed(M * 5 + N)
    CA = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8).cuda()
    CB = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8).cuda()
    SCA = (torch.rand(M, generator=g) * 5 + 0.5).cuda()
    SCB = (torch.rand(N, generator=g) * 0.1 + 0.01).cuda()
    bias = torch.randn(N, generator=g).to(dtype).cuda() if with_bias else None
    out = torch.full((M, N), float("nan"), device="cuda", dtype=dtype)
    rc = nat.lib.cbnb_b200_int8_scaled_mm(CA.data_ptr(), CB.data_ptr(), SCA.data_ptr(), SCB.data_ptr(), nat.ptr(bias),
                                          out.data_ptr(), M, N, K, 1 if dtype == torch.float16 else 2, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0  # the fused epilogue ran (100 would mean the shape was refused)
    C = (CA.double() @ CB.double().t()).to(torch.int32)  # exact: |sum| < 2^53
    want = expected_scaled_mm(C, SCA, SCB, bias, dtype)
    assert torch.equal(out.view(torch.int16), want.view(torch.int16)), \
        f"{int((out.view(torch.int16) != want.view(torch.int16)).sum())} of {out.numel()} outputs differ"


# ------------------------------------------------------------------------------------------ column-wise quantisation
def _reference_col_quant(A, threshold):
    """The reference's column half of int8_double_quant, verbatim in behaviour (backends/cuda/ops.py:262-296)."""
    absA = A.abs().view(-1, A.shape[-1])
    mask = None
    if threshold > 0.0:
        mask = absA >= threshold
        absA = absA.masked_fill(mask, 0.0)
    col_stats = absA.amax(dim=0).float()
    Ac = A.view(-1, A.shape[-1])
    if mask is not None:
        Ac = Ac.masked_fill(mask, 0.0)
    return torch.round(Ac.mul(127.0) / col_stats.unsqueeze(0)).to(torch.int8), col_stats


@pytest.mark.parametrize("shape", [(1, 8), (17, 40), (256, 1024), (1000, 777), (4096, 4096), (3, 5, 64)])
@pytest.mark.parametrize("dtype", [torch.float16])  # (the op takes fp16 only, like the reference's: its row half is fp16)
@pytest.mark.parametrize("threshold", [0.0, 3.0])
def test_native_column_quant_is_bit_identical_to_the_reference_formula(shape, dtype, threshold):
    import bitsandbytes_b200.functional as F

    g = torch.Generator(device="cpu").manual_seed(sum(shape) + int(threshold))
    A = (torch.randn(shape, generator=g) * 1.5).to(dtype).cuda()
    A.view(-1, shape[-1])[:, 0] = 0  # a column without any non-zero entry: 0 / 0 -> code 0
    if threshold > 0 and A.numel() > 64:
        A.view(-1, shape[-1])[:, 1] = 7.0  # a column made of outliers only
    want_q, want_stats = _reference_col_quant(A, threshold)
    q_row, q_col, row_stats, col_stats, outlier_cols = F.int8_double_quant(A, threshold=threshold)
    assert q_col.shape == A.shape and q_col.dtype == torch.int8 and col_stats.dtype == torch.float32
    assert torch.equal(col_stats, want_stats)
    assert torch.equal(q_col.view(-1, shape[-1]), want_q)
    # the row half is the kernel the forward uses
    rq, rs, oc = F.int8_vectorwise_quant(A, threshold=threshold)
    assert torch.equal(q_row, rq) and torch.equal(row_stats, rs)


@pytest.mark.parametrize("offset", [1, 4])
@pytest.mark.parametrize("threshold", [0.0, 3.0])
def test_native_column_quant_of_an_unaligned_view(offset, threshold):
    """A contiguous view that starts `offset` fp16 elements into its storage is not copied on its way to the column
    kernels: they must not take 16-byte loads from it."""
    import bitsandbytes_b200.functional as F

    M, K = 96, 256
    g = torch.Generator(device="cpu").manual_seed(offset + int(threshold))
    buf = (torch.randn(M * K + 8, generator=g) * 1.5).half().cuda()
    A = buf[offset:offset + M * K].view(M, K)
    assert A.is_contiguous() and A.data_ptr() % 16 != 0
    want_q, want_stats = _reference_col_quant(A, threshold)
    _, q_col, _, col_stats, _ = F.int8_double_quant(A, threshold=threshold)
    torch.cuda.synchronize()
    nat.check()
    assert torch.equal(col_stats, want_stats)
    assert torch.equal(q_col, want_q)
