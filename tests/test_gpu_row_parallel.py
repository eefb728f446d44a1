"""GPU tests of the row-parallel (input-feature-sharded) Linear4bit on one H100: the partial 4-bit GEMM (fp32
accumulators, no bias, no rounding) on every route the plain GEMM takes, the rank-order reduction, worlds of 2, 4 and 8
simulated rank by rank, the fused-pointer route under CUDA-graph capture, and the one-rank layer against matmul_4bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle
from tests import _native as nat
from tests.test_gpu_gemm4 import assert_close_to_exact, make_problem
from tests.test_gpu_gemm4_tf32 import accumulation, precision, rna_tf32, tf32_exact, ulp32  # noqa: F401

pytestmark = pytest.mark.gpu

_BF = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


def _scales(p):
    if p["absmax_8bit"] is None:
        return p["absmax"].cpu().numpy()
    return oracle.nested_absmax(p["absmax"].cpu().numpy(), p["absmax_8bit"].cpu().numpy(),
                                p["absmax_code"].cpu().numpy(), float(p["absmax_offset"].item()))


def _weights(p, dtype):
    """The decoded weights the kernels multiply by, from the CPU oracle: rn_T(value * scale) (fp32: unrounded)."""
    w = oracle.dequantize_blockwise(p["packed"].cpu().numpy(), _scales(p), p["bs"], p["N"] * p["K"], p["qt"], None,
                                    dtype)
    return nat.from_bits(w, dtype).view(p["N"], p["K"]).float()


def _partial(p, outs, ldc=None, x=None):
    from bitsandbytes_b200.backends.cuda import gemm_4bit_partial

    x = p["x"] if x is None else x
    ok = gemm_4bit_partial(x, p["packed"], (p["N"], p["K"]), p["absmax"], p["bs"], p["qt"], p["absmax_8bit"],
                           p["absmax_code"], p["absmax_offset"], outs, p["N"] if ldc is None else ldc)
    torch.cuda.synchronize()
    assert ok
    return outs


N_, K_ = 1280, 512  # ten 128-feature tiles: split-K at 16 tokens, the staged route at 4096 (16-bit)


@pytest.mark.parametrize("M", [1, 4, 8, 16, 256, 4096])
@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("nested", [False, True])
@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32", "tf32"])
def test_partial_gemm_vs_float64_oracle(precision, M, qt, nested, dtype):
    """The fp32 partial against sum_k x * W in float64 (W the exactly rounded weights of the route): half an fp32 ulp
    plus the fp32 accumulation bound of the split-K and TF32 tests."""
    precision("tf32" if dtype == "tf32" else "ieee")
    wdt = "fp32" if dtype == "tf32" else dtype
    p = make_problem(M, N_, K_, qt, wdt, nested=nested, seed=5)
    if dtype == "tf32":
        p["x"] = tf32_exact(p["x"])
    if M == 4096 and dtype in ("bf16", "fp16"):
        assert nat.lib.cbnb_b200_gemm_4bit_staged_route(M, N_, K_, 64, nat.DTYPE_ID[dtype]) == 1
    W = _weights(p, wdt)
    if dtype == "tf32" and nat.lib.cbnb_b200_gemm_4bit_path(M, N_, K_, 64, 3) == 1:
        W = rna_tf32(W)
    out = torch.full((M, N_), float("nan"), device="cuda")
    _partial(p, [out])
    y64 = p["x"].double() @ W.double().t()
    tol = 0.5 * ulp32(y64) + accumulation(K_, y64)
    assert torch.isfinite(out).all(), "unwritten outputs"
    bad = (out.double() - y64).abs() > tol
    assert not bad.any(), f"{int(bad.sum())} / {bad.numel()} off; worst {float(((out.double() - y64).abs() / tol).max()):.2f} x tol"


@pytest.mark.parametrize("M", [1, 5, 8, 16, 100, 256, 4096])
@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32"])
def test_every_destination_holds_the_same_bits(M, dtype):
    """n_outs = 4 local buffers standing in for peers, at a ragged row stride: each holds the n_outs = 1 result bit for
    bit, and nothing outside [M, N] is written."""
    p = make_problem(M, N_, K_, "nf4", dtype, seed=9)
    ldc = N_ + 3
    one = torch.full((M, ldc), float("nan"), device="cuda")
    _partial(p, [one], ldc)
    four = [torch.full((M, ldc), float("nan"), device="cuda") for _ in range(4)]
    _partial(p, four, ldc)
    nat.check()
    assert torch.isfinite(one[:, :N_]).all() and torch.isnan(one[:, N_:]).all()
    for o in four:
        assert torch.equal(o.view(torch.int32), one.view(torch.int32))


def _reduce_cpu(parts: torch.Tensor, bias, dtype):
    """The rank-order sum restated on the CPU: fp32 additions in rank order, + bias in fp32, one rounding."""
    s = parts[0].clone()
    for r in range(1, parts.shape[0]):
        s = s + parts[r]
    s = s + (bias.float() if bias is not None else torch.zeros(()))
    return s.to(dtype)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32"])
@pytest.mark.parametrize("M,N,ldc", [(1, 256, 256), (37, 520, 520), (64, 1000, 1003), (300, 96, 100)])
@pytest.mark.parametrize("with_bias", [False, True])
def test_reduce_partials_is_the_rank_order_sum(world, dtype, M, N, ldc, with_bias):
    from bitsandbytes_b200.backends.cuda import reduce_partials

    g = torch.Generator().manual_seed(world * 1000 + M + N)
    parts = torch.randn(world, M, N, generator=g) * torch.logspace(-3, 3, N)
    parts[0, 0, :4] = torch.tensor([-0.0, 0.0, 1e-30, -1e30])
    bias = torch.randn(N, generator=g).to(_BF[dtype]) if with_bias else None
    buf = torch.full((M, ldc), float("nan"), device="cuda").to(_BF[dtype])
    out = reduce_partials(parts.cuda(), _BF[dtype], bias.cuda() if bias is not None else None, out=buf[:, :N])
    torch.cuda.synchronize()
    want = _reduce_cpu(parts, bias, _BF[dtype])
    assert torch.equal(out.cpu().view(torch.int16 if dtype != "fp32" else torch.int32),
                       want.view(torch.int16 if dtype != "fp32" else torch.int32))
    assert torch.isnan(buf[:, N:].float()).all()


def _layers(qW, qs, world, bias):
    from bitsandbytes_b200.parallel import RowParallelLinear4bit, slice_quantized_weight_k

    return [RowParallelLinear4bit(slice_quantized_weight_k(qW, qs, world, r), qs.shape[1], bias) for r in range(world)]


def _simulate(layers, x, route):
    """Every rank's output, the ranks run in turn on one GPU.  stage: each partial into the rank's slot of one shared
    [w, M, N] stage (what the all-gather produces).  fused: each partial stored by the GEMM into slot r of every rank's
    own buffer, then every rank reduces its buffer."""
    from bitsandbytes_b200.backends.cuda import reduce_partials

    world = len(layers)
    K = x.shape[-1]
    xs = [x[..., L.shard.k0:L.shard.k0 + L.shard.K].contiguous() for L in layers]
    M, N = x.numel() // K, layers[0].out_features
    if route == "stage":
        stage = torch.full((world, M, N), float("nan"), device="cuda")
        for r, L in enumerate(layers):
            assert L.partial_forward(xs[r], [stage[r]])
        return [reduce_partials(stage, x.dtype, L.bias) for L in layers]
    bufs = [torch.full((world, M, N), float("nan"), device="cuda") for _ in range(world)]
    for r, L in enumerate(layers):
        assert L.partial_forward(xs[r], [b.data_ptr() + r * M * N * 4 for b in bufs])
    return [reduce_partials(bufs[r], x.dtype, L.bias) for r, L in enumerate(layers)]


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("M", [1, 8, 16, 256, 4096])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("nested,with_bias", [(False, True), (True, False)])
def test_simulated_world(world, M, dtype, nested, with_bias):
    """Fused-pointer and stage routes: the same bits on every rank and between the routes; within the oracle bound of
    the plain GEMM and close to the unsharded matmul_4bit."""
    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    N, K = 1536, 4096
    g = torch.Generator().manual_seed(world + M)
    W = (torch.randn(N, K, generator=g) / K**0.5).to(dtype).cuda()
    x = torch.randn(M, K, generator=g).to(dtype).cuda()
    bias = torch.randn(N, generator=g).to(dtype).cuda() if with_bias else None
    qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="nf4", compress_statistics=nested)
    layers = _layers(qW, qs, world, bias)
    stage = _simulate(layers, x, "stage")
    fused = _simulate(layers, x, "fused")
    torch.cuda.synchronize()
    nat.check()
    for r in range(world):
        assert torch.equal(stage[r], stage[0]) and torch.equal(fused[r], stage[0]), f"rank {r}"
    single = bnb.matmul_4bit(x, qW.t(), qs, bias=bias)
    dt = "bf16" if dtype == torch.bfloat16 else "fp16"
    Wd = F.dequantize_4bit(qW, qs).double()
    y64 = (x.double() @ Wd.t() + (bias.double() if bias is not None else 0)).cpu().numpy()
    assert_close_to_exact(stage[0], y64, dt, K)
    rel = float((stage[0].float() - single.float()).norm() / single.float().norm())
    assert rel < 2e-3


@pytest.mark.parametrize("M", [1, 4, 16, 256, 4096])
@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32", "tf32"])
@pytest.mark.parametrize("nested,with_bias", [(False, False), (False, True), (True, True)])
def test_one_rank_is_matmul_4bit_bit_for_bit(precision, M, dtype, nested, with_bias):
    """World 1 takes the partial GEMM and the reduction instead of the fused epilogue: the same bits."""
    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.parallel import RowParallelLinear4bit

    precision("tf32" if dtype == "tf32" else "ieee")
    td = torch.float32 if dtype == "tf32" else _BF[dtype]
    N, K = 1280, 1024
    g = torch.Generator().manual_seed(M)
    W = (torch.randn(N, K, generator=g) / K**0.5).to(td).cuda()
    x = torch.randn(2, M, K, generator=g).to(td).cuda()[1]
    bias = torch.randn(N, generator=g).to(td).cuda() if with_bias else None
    qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="fp4", compress_statistics=nested)
    layer = RowParallelLinear4bit.from_quantized(qW, qs, bias=bias)
    got = layer(x.view(1, M, K))
    want = bnb.matmul_4bit(x, qW.t(), qs, bias=bias)
    torch.cuda.synchronize()
    assert got.shape == (1, M, N)
    assert torch.equal(got.view(M, N), want)


def test_fused_route_replays_in_a_cuda_graph():
    """Partials stored through raw pointers into four rank buffers plus the reduction, captured once and replayed on
    new inputs: the same bits as the eager calls."""
    import bitsandbytes_b200.functional as F

    world, M, N, K = 4, 64, 2048, 4096
    g = torch.Generator().manual_seed(3)
    W = (torch.randn(N, K, generator=g) / K**0.5).to(torch.bfloat16).cuda()
    bias = torch.randn(N, generator=g).to(torch.bfloat16).cuda()
    qW, qs = F.quantize_4bit(W, quant_type="nf4")
    layers = _layers(qW, qs, world, bias)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
    static_x = x.clone()
    _simulate(layers, static_x, "fused")  # warm-up: module loads, workspace
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = _simulate(layers, static_x, "fused")
    for seed in range(3):
        static_x.copy_(torch.randn(M, K, generator=torch.Generator().manual_seed(seed)).to(torch.bfloat16).cuda())
        graph.replay()
        eager = _simulate(layers, static_x, "fused")
        torch.cuda.synchronize()
        for a, b in zip(outs, eager):
            assert torch.equal(a, b)


def test_wrapper_checks():
    from bitsandbytes_b200.backends.cuda import reduce_partials

    p = make_problem(8, 256, 128, "nf4", "bf16")
    with pytest.raises(RuntimeError):
        _partial(p, [torch.empty(8, 256, device="cuda", dtype=torch.bfloat16)])   # not fp32
    with pytest.raises(RuntimeError):
        _partial(p, [torch.empty(8 * 256 - 1, device="cuda")])                     # too small
    with pytest.raises(RuntimeError):
        _partial(p, [torch.empty(8, 256, device="cuda")] * 9)                      # more than 8 destinations
    with pytest.raises(RuntimeError):
        reduce_partials(torch.zeros(2, 4, 8, device="cuda", dtype=torch.float16), torch.float16)
    with pytest.raises(RuntimeError):
        reduce_partials(torch.zeros(2, 4, 8, device="cuda"), torch.float16, bias=torch.zeros(7, device="cuda").half())


# ------------------------------------------------------------------------------------------ processes
_SCRIPT = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import bitsandbytes_b200 as bnb
import bitsandbytes_b200.functional as F
from bitsandbytes_b200.parallel import PeerPartials, RowParallelLinear4bit, fused_forward_row
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
N, K = 2048, 7168
for M in (1, 48, 1024):
    torch.manual_seed(0)
    W = (torch.randn(N, K, device=dev) / K**0.5).to(torch.bfloat16)
    x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
    b = torch.randn(N, device=dev, dtype=torch.bfloat16)
    qW, qs = F.quantize_4bit(W, quant_type="fp4", compress_statistics=True)
    single = bnb.matmul_4bit(x, qW.t(), qs, bias=b)
    layer = RowParallelLinear4bit.from_quantized(qW, qs, bias=b, input_is_parallel=False)
    nccl = layer(x)
    peers = PeerPartials(M, N, dev)
    fused = [fused_forward_row(layer, x, peers).clone() for _ in range(3)]
    torch.cuda.synchronize()
    assert all(torch.equal(f, nccl) for f in fused), f"M={M}: fused exchange differs from the NCCL one"
    every = torch.stack([torch.empty_like(nccl) for _ in range(world)])
    dist.all_gather_into_tensor(every.view(-1), nccl.reshape(-1).contiguous())
    assert all(torch.equal(every[r], nccl) for r in range(world)), f"M={M}: ranks differ"
    if world == 1:
        assert torch.equal(nccl, single), f"M={M}: one rank differs from matmul_4bit"
    rel = float((nccl.float() - single.float()).norm() / single.float().norm())
    assert rel < 2e-3, f"M={M}: rel {rel:.2e}"
dist.barrier()
dist.destroy_process_group()
print("ROW_OK", rank)
"""


@pytest.mark.parametrize("nproc", [1, 2])
def test_processes_fused_equals_nccl(tmp_path, nproc):
    """One process per GPU: the symmetric-memory exchange and the NCCL all-gather give the same bits on every rank.
    One process checks the symmetric-memory route against matmul_4bit; two need two GPUs."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "row.py"
    script.write_text(_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29561 + nproc), str(script)],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and r.stdout.count("ROW_OK") == nproc, r.stdout[-2000:] + r.stderr[-3000:]
