"""GPU parity: blockwise quantize / dequantize through the C ABI.

Bars (BASELINE.json north_star): bit-exact quantization indices and per-block absmax,
bit-exact dequantize.  Checked against
  * the reference CUDA library built from the reference sources (oracle/_ref, same C ABI,
    same device buffers) -- strict equality;
  * the CPU oracle (oracle/oracle_c.c) -- strict equality for absmax/dequantize; for codes
    only inputs within a few ulp of a decision threshold may differ (the GPU normalises
    with the fast-math reciprocal, see oracle_c.c header);
  * size-independent properties at the BASELINE size (4 Mi elements).
"""
import numpy as np
import pytest
import torch

import oracle
from tests import _native as nat

pytestmark = pytest.mark.gpu

DTYPES = ["fp32", "bf16", "fp16"]


def _code():
    from bitsandbytes_b200.functional import create_dynamic_map

    return create_dynamic_map().cuda()


def _inputs(n, dtype, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(1234 + n)
    a = (torch.randn(n, generator=g) * scale).to(nat.DTYPE[dtype])
    if n > 10:
        a[3] = 0
        a[7] = -a.abs().max()  # an exact -absmax element
    return a.cuda()


# ---------------------------------------------------------------------------- dequantize
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("qt", [None, "nf4", "fp4"])
@pytest.mark.parametrize("n,bs", [(4096 * 3, 4096), (64 * 100, 64), (8192 + 37, 256), (1001, 128), (96, 32), (7, 64)])
def test_dequantize_matches_oracle_and_reference(dtype, qt, n, bs):
    # the reference's 8-bit kernels take blocksize >= 64: below that only the oracle is compared
    ref_ok = not (qt is None and bs < 64)
    g = torch.Generator(device="cpu").manual_seed(n + bs)
    nbytes = n if qt is None else (n + 1) // 2
    codes = torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8).cuda()
    absmax = (torch.rand(-(n // -bs), generator=g) * 4 + 1e-3).cuda()
    code = _code() if qt is None else None
    got = nat.dequantize(nat.lib, codes, absmax, bs, n, qt, code, dtype)
    nat.check()
    want = oracle.dequantize_blockwise(codes.cpu().numpy(), absmax.cpu().numpy(), bs, n, qt,
                                       None if code is None else code.cpu().numpy(), dtype)
    g_bits = nat.to_bits(got)
    if dtype == "fp32":
        np.testing.assert_array_equal(g_bits.view(np.uint32), want.view(np.uint32))
    else:
        np.testing.assert_array_equal(g_bits, want)
    ref = nat.ref_cuda() if ref_ok else None
    if ref is not None:
        r = nat.dequantize(ref, codes, absmax, bs, n, qt, code, dtype)
        assert torch.equal(got.view(torch.int32 if dtype == "fp32" else torch.int16),
                           r.view(torch.int32 if dtype == "fp32" else torch.int16))


def test_dequantize_unaligned_output_pointer():
    n, bs = 4096, 64
    codes = torch.randint(0, 256, (n // 2,), dtype=torch.uint8).cuda()
    absmax = torch.rand(n // bs).cuda() + 0.1
    buf = torch.zeros(n + 8, device="cuda", dtype=torch.bfloat16)
    out = buf[1:n + 1]  # 2-byte aligned only
    nat.lib.cdequantize_blockwise_bf16_nf4(None, codes.data_ptr(), absmax.data_ptr(), out.data_ptr(), bs, n, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    want = oracle.dequantize_blockwise(codes.cpu().numpy(), absmax.cpu().numpy(), bs, n, "nf4", None, "bf16")
    np.testing.assert_array_equal(nat.to_bits(out), want)


# ---------------------------------------------------------------------------- quantize
def _check_codes_vs_oracle(A_f32, got_codes, got_absmax, bs, qt, code):
    q, absmax = oracle.quantize_blockwise(A_f32, bs, qt, code)
    np.testing.assert_array_equal(got_absmax, absmax)
    bad = np.nonzero(got_codes != q)[0]
    n = A_f32.size
    assert bad.size <= max(2, n // 1000), f"{bad.size} code mismatches vs the CPU oracle"
    for b in bad[:64]:
        elems = [b] if qt is None else [2 * b, 2 * b + 1]
        for e in elems:
            if e >= n:
                continue
            x = np.float32(A_f32[e]) * (np.float32(1.0) / absmax[e // bs])
            if qt is None:
                bounds = (code[:-1].astype(np.float64) + code[1:].astype(np.float64)) / 2
                d = np.min(np.abs(np.float64(x) - bounds))
            else:
                fn = oracle.lib().oracle_nf4_threshold_distance if qt == "nf4" else oracle.lib().oracle_fp4_threshold_distance
                d = fn(float(x))
            gq = got_codes[b] if qt is None else ((got_codes[b] >> 4) if e % 2 == 0 else (got_codes[b] & 15))
            oq = q[b] if qt is None else ((q[b] >> 4) if e % 2 == 0 else (q[b] & 15))
            if gq != oq:
                assert d <= 8 * np.spacing(np.float32(max(abs(x), 1e-3))), (e, x, gq, oq, d)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("qt", [None, "nf4", "fp4"])
@pytest.mark.parametrize("n,bs", [(4096 * 5, 4096), (4096 * 4, 64), (4096 * 2 + 777, 256), (4096 + 1, 2048),
                                  (999, 128), (64 * 3, 32), (5, 64), (4096 * 3, 512), (4096 * 2, 1024)])
def test_quantize_bit_exact(dtype, qt, n, bs):
    # the reference's 8-bit kernels take blocksize >= 64: below that only the oracle is compared
    ref_ok = not (qt is None and bs < 64)
    A = _inputs(n, dtype)
    code = _code() if qt is None else None
    got_q, got_absmax = nat.quantize(nat.lib, A, bs, qt, code, dtype)
    nat.check()
    ref = nat.ref_cuda() if ref_ok else None
    if ref is not None:
        ref_q, ref_absmax = nat.quantize(ref, A, bs, qt, code, dtype)
        assert torch.equal(got_absmax, ref_absmax), "absmax differs from the reference CUDA kernel"
        neq = (got_q != ref_q).sum().item()
        assert neq == 0, f"{neq} codes differ from the reference CUDA kernel"
    _check_codes_vs_oracle(A.float().cpu().numpy(), got_q.cpu().numpy(), got_absmax.cpu().numpy(), bs, qt,
                           None if code is None else code.cpu().numpy())


def test_quantize_all_zero_block_and_constant_block():
    # all-zero block: 0 * rcp(0) = NaN -> every comparison false (reference kernels.cu:114-152)
    A = torch.randn(256, device="cuda")
    A[64:128] = 0
    A[128:192] = 3.0
    for qt in ("nf4", "fp4", None):
        code = _code() if qt is None else None
        q, absmax = nat.quantize(nat.lib, A, 64, qt, code, "fp32")
        nat.check()
        assert absmax[1].item() == 0.0 and absmax[2].item() == 3.0
        ref = nat.ref_cuda()
        if ref is not None:
            rq, rabs = nat.quantize(ref, A, 64, qt, code, "fp32")
            assert torch.equal(q, rq) and torch.equal(absmax, rabs)
        if qt == "nf4":
            assert torch.all(q[32:64] == 0x00) and torch.all(q[64:96] == 0xFF)


def test_stream_taking_quantize_matches_default_stream_entry():
    A = _inputs(4096 * 3, "bf16")
    q0, a0 = nat.quantize(nat.lib, A, 64, "nf4", None, "bf16")
    q1 = torch.zeros_like(q0)
    a1 = torch.zeros_like(a0)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        nat.lib.cbnb_b200_quantize_blockwise(None, A.data_ptr(), a1.data_ptr(), q1.data_ptr(), 64, A.numel(), 2, 2,
                                             s.cuda_stream)
    s.synchronize()
    nat.check()
    assert torch.equal(q0, q1) and torch.equal(a0, a1)


# ---------------------------------------------------------------------------- BASELINE size
@pytest.mark.parametrize("bs", [4096, 256])
def test_c1_size_properties(bs):
    """C1: 4 Mi fp32 elements.  absmax == blockwise max|x|, round trip error bounded by the
    reference's own test bounds (reference tests/test_functional.py:113-169), codes monotone in x
    inside every block (sortedness), |dequantized| <= absmax."""
    n = 4 * 1024 * 1024
    A = torch.randn(n, device="cuda")
    code = _code()
    q, absmax = nat.quantize(nat.lib, A, bs, None, code, "fp32")
    nat.check()
    assert torch.equal(absmax, A.view(-1, bs).abs().amax(dim=1))
    D = nat.dequantize(nat.lib, q, absmax, bs, n, None, code, "fp32")
    err = (A - D).abs()
    assert err.mean().item() < 0.011
    assert (err / (A.abs() + 1e-8)).mean().item() < 0.018
    # sortedness: within a block, x_i <= x_j implies code_i <= code_j (the map is ascending)
    order = A.view(-1, bs).argsort(dim=1)
    qs = torch.gather(q.view(-1, bs).to(torch.int16), 1, order)
    assert (qs[:, 1:] >= qs[:, :-1]).all()
    # and the dequantized values never exceed the block's absmax
    assert (D.view(-1, bs).abs() <= absmax.view(-1, 1)).all()
    ref = nat.ref_cuda()
    if ref is not None:
        rq, rabs = nat.quantize(ref, A, bs, None, code, "fp32")
        assert torch.equal(rabs, absmax)
        assert (rq != q).sum().item() == 0


@pytest.mark.parametrize("qt", ["nf4", "fp4"])
def test_c2_weight_quantize_properties(qt):
    """4096x4096 bf16 weight, blocksize 64: mean abs round-trip error inside the reference's
    published table (reference tests/test_functional.py:606-651: NF4 0.072798, FP4 0.096543,
    both +- a few 1e-4) and bit-equality with the reference CUDA kernel."""
    W = torch.randn(4096, 4096, device="cuda", dtype=torch.bfloat16)
    q, absmax = nat.quantize(nat.lib, W.view(-1), 64, qt, None, "bf16")
    nat.check()
    D = nat.dequantize(nat.lib, q, absmax, 64, W.numel(), qt, None, "bf16")
    err = (W.float().view(-1) - D.float()).abs().mean().item()
    lo, hi = (0.0715, 0.0742) if qt == "nf4" else (0.0950, 0.0985)
    assert lo < err < hi, err
    ref = nat.ref_cuda()
    if ref is not None:
        rq, rabs = nat.quantize(ref, W.view(-1), 64, qt, None, "bf16")
        assert torch.equal(rabs, absmax) and torch.equal(rq, q)
