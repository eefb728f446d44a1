"""GPU parity at BASELINE.json's FULL sizes (round-1 review: C3 and C4 were only covered at toy sizes).

* configs[2]  the whole LLM.int8() forward (row quantise -> int8 GEMM -> dequantise -> outlier columns) at
              4096 x 11008, M = 4096, threshold 6.0 with 0 / 5 / 41 outlier columns, through the public API,
              against the REFERENCE CUDA library's chain on the same buffers (cint8_vector_quant -> cigemmlt_32 ->
              cdequant_mm_int32_fp16: bit for bit) plus an fp64 outlier term.
* configs[3]  FP4 + double quant at the column shard of the 70B layer (3584 x 8192), M in {1, 16, 256, 4096}:
              fused GEMM vs (bit-exact dequantize) @ x in fp32, vs the CPU oracle on a sampled sub-problem and vs
              the reference CUDA library's own fused kernel.
* the fused outlier epilogue against an explicit chain at small ragged shapes; one process driving two devices;
  a 2-GPU run where the fused peer-store gather == NCCL gather (bit-exact) ~= single-GPU result (skipped on one GPU).
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle
from tests import _native as nat
from tests.test_gpu_gemm4 import assert_close_to_exact, exact, make_problem, run

pytestmark = pytest.mark.gpu


def _ulp16(x: torch.Tensor, dtype) -> torch.Tensor:
    mant = 10 if dtype == torch.float16 else 7
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0**-24 if dtype == torch.float16 else 1e-38)))
    if dtype == torch.float16:
        e = e.clamp_min(-14)
    return torch.exp2(e - mant)


# ------------------------------------------------------------------------------------------ fused outlier epilogue
@pytest.mark.parametrize("M,N,K,J", [(9, 24, 64, 1), (130, 300, 192, 5), (257, 1000, 1024, 8), (64, 512, 256, 9),
                                     (300, 384, 512, 41), (128, 256, 128, 64)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("with_bias", [False, True])
def test_fused_mixed_mm_equals_the_explicit_chain(M, N, K, J, dtype, with_bias):
    """cbnb_b200_int8_mixed_mm == T( float(T(int8 part incl. bias)) + sum_j subA * subBT ): the int8 part must be
    bit-identical to the unfused kernel, the outlier sum may differ from an fp64 sum only by fp32 accumulation."""
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N + J)
    CA = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8).cuda()
    CB = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8).cuda()
    SCA = (torch.rand(M, generator=g) * 5 + 0.5).cuda()
    SCB = (torch.rand(N, generator=g) * 0.1 + 0.01).cuda()
    bias = torch.randn(N, generator=g).to(dtype).cuda() if with_bias else None
    A = (torch.randn(M, K, generator=g) * 2).to(dtype).cuda()
    cols = torch.randperm(K, generator=g)[:J].sort().values.cuda()
    A[:, cols] = (torch.randn(M, J, generator=g) * 4 + 9).to(dtype).cuda()
    CA[:, cols] = 0
    did = 1 if dtype == torch.float16 else 2
    jpad = -(-J // 8) * 8
    subA = torch.full((M, jpad), float("nan"), device="cuda", dtype=dtype)
    subBT = torch.full((N, jpad), float("nan"), device="cuda", dtype=dtype)
    nat.lib.cbnb_b200_int8_outlier_prep(A.data_ptr(), CB.data_ptr(), SCB.data_ptr(), cols.data_ptr(), J, jpad, M, N, K, did,
                                        subA.data_ptr(), subBT.data_ptr(), nat.stream())
    torch.cuda.synchronize()
    nat.check()
    # the two operands: gathered activations, and CB * SCB * (1/127) in fp32 rounded to T (reference _ops.py:118-121)
    assert torch.equal(subA[:, :J], A[:, cols]) and (subA[:, J:] == 0).all()
    want_b = (CB[:, cols].float() * SCB.view(-1, 1) * 7.874015718698502e-3).to(dtype)
    assert torch.equal(subBT[:, :J], want_b) and (subBT[:, J:] == 0).all()

    out = torch.full((M, N), float("nan"), device="cuda", dtype=dtype)
    rc = nat.lib.cbnb_b200_int8_mixed_mm(CA.data_ptr(), CB.data_ptr(), SCA.data_ptr(), SCB.data_ptr(), nat.ptr(bias),
                                         subA.data_ptr(), subBT.data_ptr(), jpad, out.data_ptr(), M, N, K, did, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    base = torch.zeros_like(out)
    rc = nat.lib.cbnb_b200_int8_scaled_mm(CA.data_ptr(), CB.data_ptr(), SCA.data_ptr(), SCB.data_ptr(), nat.ptr(bias),
                                          base.data_ptr(), M, N, K, did, nat.stream())
    torch.cuda.synchronize()
    assert rc == 0
    o64 = subA[:, :J].double() @ subBT[:, :J].double().t()
    exact64 = base.double() + o64
    want = exact64.to(dtype)
    diff = (out.double() - exact64).abs()
    tol = 0.5 * _ulp16(exact64, dtype).double() * 1.001 + 2.0**-21 * (1 + o64.abs()) * J**0.5
    assert (diff <= tol).all(), f"{int((diff > tol).sum())} outputs off, worst excess {(diff - tol).max().item():.3e}"
    assert (out != want).float().mean().item() < 2e-3  # only fp32-vs-fp64 rounding-boundary flips


# ------------------------------------------------------------------------------------------ configs[2] at full size
@pytest.mark.parametrize("n_outliers", [0, 5, 41])
def test_llm_int8_forward_c3_vs_reference_cuda_chain(n_outliers):
    import bitsandbytes_b200 as bnb

    ref = nat.ref_cuda()
    K, N, M = 4096, 11008, 4096
    g = torch.Generator(device="cpu").manual_seed(41 + n_outliers)
    lin = torch.nn.Linear(K, N, bias=True)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(N, K, generator=g) * 0.02)
        lin.bias.copy_(torch.randn(N, generator=g) * 0.1)
    layer = bnb.nn.Linear8bitLt(K, N, bias=True, has_fp16_weights=False, threshold=6.0)
    layer.load_state_dict(lin.state_dict())
    layer = layer.to("cuda").eval()
    x = torch.randn(M, K, generator=g).clamp_(-5.5, 5.5).to(torch.float16).cuda()
    cols = torch.randperm(K, generator=g)[:n_outliers].sort().values.cuda()
    if n_outliers:
        x[:, cols] = (torch.randn(M, n_outliers, generator=g) * 3).abs().add_(6.5).to(torch.float16).cuda()
        x[::7, cols[0]] = 0.25  # a column is an outlier column as soon as ONE row crosses the threshold
    with torch.no_grad():
        y = layer(x)
    torch.cuda.synchronize()
    nat.check()
    assert y.dtype == torch.float16 and y.shape == (M, N)
    if n_outliers:
        assert torch.equal(layer.state.idx.sort().values, cols)
    CB, SCB = layer.state.CB, layer.state.SCB
    bias16 = layer.bias.to(torch.float16).contiguous()

    # ---- the reference CUDA library's chain on the same inputs
    rq = torch.zeros(M, K, device="cuda", dtype=torch.int8)
    rstats = torch.zeros(M, device="cuda")
    ref.cint8_vector_quant(x.data_ptr(), rq.data_ptr(), rstats.data_ptr(), 6.0, M, K, nat.stream())
    torch.cuda.synchronize()
    if n_outliers:
        rq[:, cols] = 0  # reference backends/cuda/ops.py:233-236
    # weights: the reference's row quantisation of the fp16 weight must give the CB / SCB our module holds
    wq = torch.zeros(N, K, device="cuda", dtype=torch.int8)
    wstats = torch.zeros(N, device="cuda")
    w16 = lin.weight.detach().to("cuda", torch.float16).contiguous()
    ref.cint8_vector_quant(w16.data_ptr(), wq.data_ptr(), wstats.data_ptr(), 0.0, N, K, nat.stream())
    torch.cuda.synchronize()
    assert torch.equal(wq, CB) and torch.equal(wstats, SCB)
    acc = torch.zeros(M, N, device="cuda", dtype=torch.int32)
    rc = ref.cigemmlt_32(ref.get_context(), N, M, K, wq.data_ptr(), rq.data_ptr(), acc.data_ptr(), None, K, K, N, nat.stream())
    torch.cuda.synchronize()
    if rc != 0:
        # the reference's cublasLt call rejects this shape on this CUDA build (status 7 in round 2's run): the int8
        # GEMM is exact integer arithmetic, so any exact engine gives the accumulators the reference would produce
        acc = torch._int_mm(rq, wq.t())
    # exactness on a row sample, whichever engine produced `acc`
    rows = torch.arange(0, M, 257, device="cuda")
    assert torch.equal(acc[rows], (rq[rows].double() @ wq.double().t()).to(torch.int32))
    r16 = torch.zeros(M, N, device="cuda", dtype=torch.float16)
    ref.cdequant_mm_int32_fp16(acc.data_ptr(), rstats.data_ptr(), wstats.data_ptr(), r16.data_ptr(), bias16.data_ptr(), M, N,
                               nat.stream())
    torch.cuda.synchronize()
    if n_outliers == 0:
        assert torch.equal(y.view(torch.int16), r16.view(torch.int16)), "LLM.int8() forward differs from the reference chain"
        return
    subA = x[:, cols]
    subB = (wq[:, cols].float() * wstats.view(-1, 1) * 7.874015718698502e-3).to(torch.float16)
    o64 = subA.double() @ subB.double().t()
    exact64 = r16.double() + o64
    diff = (y.double() - exact64).abs()
    tol = 0.5 * _ulp16(exact64, torch.float16).double() * 1.001 + 2.0**-21 * (1 + o64.abs()) * n_outliers**0.5
    assert (diff <= tol).all(), f"{int((diff > tol).sum())} outputs off, worst excess {(diff - tol).max().item():.3e}"
    assert (y != exact64.to(torch.float16)).float().mean().item() < 2e-3
    # and the reference's own second step (cuBLAS addmm on the fp16 tensor) agrees to within one rounding
    ref_out = r16.addmm(subA, subB.t())
    assert (y.float() - ref_out.float()).abs().max().item() <= 2 * _ulp16(exact64, torch.float16).max().item()


# ------------------------------------------------------------------------------------------ configs[3] shard shape
@pytest.mark.parametrize("M", [1, 16, 256, 4096])
def test_fp4_double_quant_at_the_c4_shard_shape(M):
    """One rank's shard of the 8192 -> 28672 layer (28672 / 8 = 3584 rows, K = 8192), FP4 + double quant."""
    N, K = 3584, 8192
    p = make_problem(M, N, K, "fp4", "bf16", nested=True, seed=17)
    got = run(nat.lib, p)
    nat.check()
    # (1) fused == (bit-exact dequantize, nested scales resolved as F.dequantize_4bit does) @ x, fp32 accumulate
    from bitsandbytes_b200.functional import QuantState, dequantize_4bit, dequantize_blockwise

    state2 = QuantState(absmax=p["absmax"], code=p["absmax_code"], blocksize=256, dtype=torch.float32)
    absmax = dequantize_blockwise(p["absmax_8bit"], state2) + p["absmax_offset"]
    qs = QuantState(absmax=absmax, shape=torch.Size([N, K]), dtype=torch.bfloat16, blocksize=64, quant_type="fp4")
    W = dequantize_4bit(p["packed"].view(-1, 1), qs)
    want32 = p["x"].float() @ W.float().t()
    diff = (got.float() - want32).abs()
    tol = want32.abs() * (2.0**-8 * 1.01) + 2.0**-20 * (K**0.5) * (1 + want32.abs())
    assert (diff <= tol).all(), f"max excess {(diff - tol).max().item():.3e}"
    rel = (got.float() - want32.to(torch.bfloat16).float()).norm() / want32.norm()
    assert rel.item() <= 1e-3
    # (2) the CPU oracle (double accumulation) on a sub-problem: the first 64 features of 8 token rows
    ms = min(M, 8)
    sub = dict(p, M=ms, N=64, x=p["x"][:ms].contiguous(), packed=p["packed"][: 64 * K // 2].contiguous(),
               absmax_8bit=p["absmax_8bit"][: 64 * K // 64].contiguous(), bias=None)
    assert_close_to_exact(got[:ms, :64].contiguous(), exact(sub), "bf16", K)
    # (3) the reference CUDA library's fused kernel on the same buffers (double-quant arguments included)
    ref = nat.ref_cuda()
    r = run(ref, p)
    if M <= 3:  # its SIMT kernel rounds every product to bf16: compare error against the fp32 product instead
        assert (got.float() - want32).norm() <= (r.float() - want32).norm() * 1.05 + 1e-6
    else:
        rel_ref = (got.float() - r.float()).norm() / r.float().norm()
        assert rel_ref.item() <= 1e-3, rel_ref.item()


# ------------------------------------------------------------------------------------------ tensor-core kernel, large M
@pytest.mark.parametrize("M,N,K,qt,dtype,kw", [
    (512, 256, 128, "nf4", "bf16", {}), (600, 512, 320, "fp4", "fp16", dict(bias=True)),
    (513, 384, 192, "nf4", "bf16", dict(nested=True)), (1000, 1024, 1024, "nf4", "bf16", {}),
    (777, 1000, 704, "nf4", "bf16", dict(bs=32, bias=True)), (640, 768, 512, "fp4", "bf16", dict(bs=128, nested=True)),
    (2048, 2304, 2048, "nf4", "bf16", dict(bias=True)),
])
def test_pair_kernel_vs_oracle_and_one_cta_kernel(M, N, K, qt, dtype, kw):
    """The wgmma kernel at large M (every token tile, with and without a forced K split) against the
    double-precision oracle, and -- without a split, where the fp32 summation order is the same -- bit for bit
    across token tiles."""
    p = make_problem(M, N, K, qt, dtype, **kw)
    y64 = exact(p) if M * N * K <= 2**31 else None
    nat.lib.cbnb_b200_gemm_4bit_force_path(1)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kblocks = -(-K // 128)

    def splits_of(mt, sp):
        """(splits the launcher makes of a forced sp, whether it serves them): >= one 128-deep stage per split, and
        a split grid must be one co-resident wave (one CTA per SM)"""
        v = min(sp, kblocks, 16)
        per = -(-kblocks // v)
        s = -(-kblocks // per)
        return s, s == 1 or -(-N // 128) * -(-M // mt) * s <= sms

    base = None
    ran_split = False
    for mt in (32, 64, 128):
        for sp in (1, 2, 3):
            s, served = splits_of(mt, sp)
            out = torch.full((M, N), float("nan"), device="cuda", dtype=nat.DTYPE[dtype])
            rc = nat.lib.cbnb_b200_gemm_4bit_pair(
                nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
                nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]), nat.ptr(out), nat.ptr(p["bias"]), M, N, K, N, p["bs"],
                nat.QT_ID[qt], nat.DTYPE_ID[dtype], mt, sp, None, nat.stream())
            torch.cuda.synchronize()
            nat.check()
            if not served:
                assert rc == 100, (mt, sp)  # the splits of a tile wait for each other: refused, not run
                continue
            assert rc == 0, (mt, sp)
            ran_split |= s > 1
            if y64 is not None:
                assert_close_to_exact(out, y64, dtype, K)
            if sp == 1:
                if base is None:
                    base = out
                assert torch.equal(out.view(torch.int16), base.view(torch.int16)), f"mt={mt}: token tiles disagree"
    nat.lib.cbnb_b200_gemm_4bit_force_path(-1)
    # a split ran, unless K is one stage or even the widest token tile's grid, split in two, exceeds one wave
    if kblocks > 1 and -(-N // 128) * -(-M // 128) * 2 <= sms:
        assert ran_split
    if y64 is None:
        W = nat.dequantize(nat.lib, p["packed"], p["absmax"], p["bs"], N * K, qt, None, dtype).view(N, K)
        want = p["x"].float() @ W.float().t() + (p["bias"].float() if p["bias"] is not None else 0)
        assert ((base.float() - want).norm() / want.norm()).item() < 2e-3


def test_pair_kernel_multi_destination_tma_stores():
    """The fused all-gather epilogue of the tensor-core kernel at large M on one GPU: three destination buffers
    receive this shard's columns of a wider output; nothing else is touched; M tail and N tail."""
    import ctypes as ct

    M, N, K, NF = 1100, 320, 512, 1024
    p = make_problem(M, N, K, "nf4", "bf16", bias=True, seed=21)
    want = run(nat.lib, p)
    bufs = [torch.full((M, NF), -7.0, dtype=torch.bfloat16, device="cuda") for _ in range(3)]
    col0 = 384
    ptrs = (ct.c_void_p * 3)(*[b.data_ptr() + col0 * 2 for b in bufs])
    rc = nat.lib.cbnb_b200_gemm_4bit_multi_out(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), None, None, None, ct.cast(ptrs, ct.c_void_p), 3,
        nat.ptr(p["bias"]), M, N, K, NF, p["bs"], nat.QT_ID["nf4"], 2, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0
    for b in bufs:
        assert torch.equal(b[:, col0:col0 + N], want)
        assert (b[:, :col0] == -7.0).all() and (b[:, col0 + N:] == -7.0).all()
    # an output whose row pitch is not a multiple of 16 bytes: same result
    odd = torch.full((M, N + 3), -7.0, dtype=torch.bfloat16, device="cuda")
    nat.lib.cbnb_b200_gemm_4bit_strided(nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), None, None, None,
                                        odd.data_ptr(), nat.ptr(p["bias"]), M, N, K, N + 3, p["bs"], nat.QT_ID["nf4"], 2,
                                        nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert torch.equal(odd[:, :N], want) and (odd[:, N:] == -7.0).all()


# ------------------------------------------------------------------------------------------ several devices, one process
def test_one_process_drives_two_devices():
    """The shared-memory opt-in and the launch state are per device (reference csrc/gemm_4bit.cu:18-36 keeps
    16-entry per-device caches for the same reason): HF device_map="auto" runs layers on cuda:1 after cuda:0."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    outs = []
    for dev in ("cuda:0", "cuda:1", "cuda:0"):
        torch.manual_seed(0)
        W = (torch.randn(512, 1024) / 32).to(torch.bfloat16).to(dev)
        x = torch.randn(700, 1024).to(torch.bfloat16).to(dev)
        qW, qs = F.quantize_4bit(W, quant_type="nf4")
        y_big = bnb.matmul_4bit(x, qW.t(), qs)          # wgmma kernel, 128-token tiles
        y_mid = bnb.matmul_4bit(x[:100], qW.t(), qs)    # wgmma kernel, one token tile
        y_small = bnb.matmul_4bit(x[:24], qW.t(), qs)   # split-K
        A8 = torch.randint(-127, 128, (300, 1024), dtype=torch.int8, device=dev)
        B8 = torch.randint(-127, 128, (256, 1024), dtype=torch.int8, device=dev)
        C = F.int8_linear_matmul(A8, B8)
        assert torch.equal(C, (A8.double() @ B8.double().t()).to(torch.int32))
        torch.cuda.synchronize(dev)
        outs.append((y_big.cpu(), y_mid.cpu(), y_small.cpu()))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    for a, b in zip(outs[0], outs[2]):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------ 2 GPUs
_TWO_GPU_SCRIPT = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import bitsandbytes_b200 as bnb
import bitsandbytes_b200.functional as F
from bitsandbytes_b200.parallel import ColumnParallelLinear4bit, PeerGather, fused_forward, slice_quantized_weight
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
N, K = 7168, 2048
for M in (48, 1024):
    torch.manual_seed(0)
    W = (torch.randn(N, K, device=dev) / K**0.5).to(torch.bfloat16)
    x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
    qW, qs = F.quantize_4bit(W, quant_type="fp4", compress_statistics=True)
    single = bnb.matmul_4bit(x, qW.t(), qs)
    layer = ColumnParallelLinear4bit(slice_quantized_weight(qW, qs, world, rank), N)
    nccl = layer(x).reshape(M, N)
    peers = PeerGather(M, N, torch.bfloat16, dev)
    fused = fused_forward(layer, x, peers).clone()
    torch.cuda.synchronize()
    # the fused exchange must be BIT-identical to the NCCL one (same kernel, same shard shapes); against the
    # single-GPU layer the K split of the partial last round differs with the tile count, so only the fp32
    # summation order -- at most an ulp of bf16 per element -- may differ
    assert torch.equal(fused, nccl), f"M={M}: fused peer-store gather differs from the NCCL gather"
    rel = float((nccl.float() - single.float()).norm() / single.float().norm())
    assert rel < 2e-3 and not torch.isnan(nccl.float()).any(), f"M={M}: sharded result off the single-GPU one (rel {rel:.2e})"
    worst = float((nccl.float() - single.float()).abs().max() / single.float().abs().max())
    assert worst < 1e-2, f"M={M}: max deviation {worst:.2e}"
dist.barrier()
dist.destroy_process_group()
print("TWO_GPU_OK", rank)
"""


def test_two_gpu_fused_gather_equals_nccl_equals_single_gpu(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    script = tmp_path / "two_gpu.py"
    script.write_text(_TWO_GPU_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29541", str(script)],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and r.stdout.count("TWO_GPU_OK") == 2, r.stdout[-2000:] + r.stderr[-3000:]
