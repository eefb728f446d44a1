"""GPU tests of the sequence-parallel Linear4bit layers on one H100: the scatter partial GEMM against the broadcast one on
every route the dispatch takes, worlds of 2, 4 and 8 simulated rank by rank for the row and column layers and an MLP
chain, a CUDA-graph replay of the fused routes, and the one- / two-process symmetric-memory runs."""
import os
import subprocess
import sys

import pytest
import torch

from tests import _native as nat
from tests.test_gpu_gemm4 import make_problem
from tests.test_gpu_gemm4_tf32 import precision, tf32_exact  # noqa: F401

pytestmark = pytest.mark.gpu

_DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32, "tf32": torch.float32}
N_, K_ = 1280, 512  # ten 128-feature tiles: split-K at 16 tokens, the staged route at 4096 (16-bit)


def _call(fn, p, outs, ldc):
    ok = fn(p["x"], p["packed"], (p["N"], p["K"]), p["absmax"], p["bs"], p["qt"], p["absmax_8bit"], p["absmax_code"],
            p["absmax_offset"], outs, ldc)
    torch.cuda.synchronize()
    assert ok
    nat.check()


def _route(M, dtype):
    did = {"fp32": 0, "fp16": 1, "bf16": 2, "tf32": 3}[dtype]
    return nat.lib.cbnb_b200_gemm_4bit_path(M, N_, K_, 64, did), nat.lib.cbnb_b200_gemm_4bit_staged_route(M, N_, K_, 64,
                                                                                                          did)


_CASES = [(w, M) for w in (1, 2, 4, 8) for M in (1, 2, 4, 8, 16, 256, 4096) if M % w == 0 and (M > 1 or w == 1)]


@pytest.mark.parametrize("world,M", _CASES)
@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("nested", [False, True])
@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32", "tf32"])
def test_scatter_equals_broadcast(precision, world, M, qt, nested, dtype):
    """The scatter destinations, stacked, hold the one-destination partial bit for bit, and nothing is written outside
    each destination's rows or past N at a ragged row stride."""
    from bitsandbytes_b200.backends.cuda import gemm_4bit_partial, gemm_4bit_partial_scatter

    precision("tf32" if dtype == "tf32" else "ieee")
    p = make_problem(M, N_, K_, qt, "fp32" if dtype == "tf32" else dtype, nested=nested, seed=11)
    if dtype == "tf32":
        p["x"] = tf32_exact(p["x"])
    path, staged = _route(M, dtype)
    if dtype in ("bf16", "fp16"):
        # M <= 8: the CUDA-core GEMV or the mma.sync decode kernel; 16: the wgmma kernel split along K (10 tiles);
        # 4096: the staged route
        assert path == (1 if M >= 16 else path) and path in (0, 1, 3) and staged == (M == 4096)
    if dtype == "fp32":
        assert path in (0, 2)  # the CUDA-core kernels
    ldc = N_ + 3
    one = torch.full((M, ldc), float("nan"), device="cuda")
    _call(gemm_4bit_partial, p, [one], ldc)
    Ms = M // world
    outs = [torch.full((Ms + 1, ldc), float("nan"), device="cuda") for _ in range(world)]
    _call(gemm_4bit_partial_scatter, p, [o[:Ms] for o in outs], ldc)
    got = torch.cat([o[:Ms] for o in outs])
    assert torch.equal(got.view(torch.int32), one.view(torch.int32))
    assert torch.isfinite(got[:, :N_]).all() and torch.isnan(got[:, N_:]).all()
    assert all(torch.isnan(o[Ms]).all() for o in outs), "a row past a destination's share was written"


def _quantized(N, K, dtype, nested, seed, qt="nf4"):
    import bitsandbytes_b200.functional as F

    g = torch.Generator().manual_seed(seed)
    W = (torch.randn(N, K, generator=g) / K**0.5).to(dtype).cuda()
    return F.quantize_4bit(W, blocksize=64, quant_type=qt, compress_statistics=nested)


def _row_layers(qW, qs, world, bias, sp):
    from bitsandbytes_b200.parallel import RowParallelLinear4bit, slice_quantized_weight_k

    return [RowParallelLinear4bit(slice_quantized_weight_k(qW, qs, world, r), qs.shape[1], bias, sequence_parallel=sp)
            for r in range(world)]


def _row_sp(layers, x, route):
    """Every rank's SP output, the ranks run in turn.  stage: each rank's full partial, chunk s sent to rank s (what
    the all-to-all produces).  fused: the scatter GEMM stores rank s's rows into slot r of rank s's buffer."""
    from bitsandbytes_b200.backends.cuda import reduce_partials

    world = len(layers)
    K = x.shape[-1]
    xs = [x[..., L.shard.k0:L.shard.k0 + L.shard.K].contiguous() for L in layers]
    M, N = x.numel() // K, layers[0].out_features
    Ms = M // world
    bufs = [torch.full((world, Ms, N), float("nan"), device="cuda") for _ in range(world)]
    for r, L in enumerate(layers):
        if route == "stage":
            send = torch.full((world, Ms, N), float("nan"), device="cuda")
            assert L.partial_forward(xs[r], [send])
            for s in range(world):
                bufs[s][r].copy_(send[s])
        else:
            assert L.partial_scatter(xs[r], [b.data_ptr() + r * Ms * N * 4 for b in bufs])
    lead = (x.shape[0] // world, *x.shape[1:-1], N)
    return [reduce_partials(bufs[r], x.dtype, L.bias).view(lead) for r, L in enumerate(layers)]


def _row_full(layers, x):
    """The non-SP output (every rank holds the same): the partials of all ranks reduced in rank order."""
    from bitsandbytes_b200.backends.cuda import reduce_partials

    K = x.shape[-1]
    M, N = x.numel() // K, layers[0].out_features
    stage = torch.full((len(layers), M, N), float("nan"), device="cuda")
    for r, L in enumerate(layers):
        assert L.partial_forward(x[..., L.shard.k0:L.shard.k0 + L.shard.K].contiguous(), [stage[r]])
    return reduce_partials(stage, x.dtype, layers[0].bias).view(*x.shape[:-1], N)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("M", [8, 16, 256, 4096])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("nested,with_bias", [(False, True), (True, False)])
def test_row_layer_sp_is_the_token_slice(world, M, dtype, nested, with_bias):
    N, K = 1536, 4096
    qW, qs = _quantized(N, K, dtype, nested, world + M)
    g = torch.Generator().manual_seed(M)
    b = 2 if (M // 2) % world == 0 else 1
    x = torch.randn(M // b, b, K, generator=g).to(dtype).cuda()  # [s, b, h]: tokens split along s
    bias = torch.randn(N, generator=g).to(dtype).cuda() if with_bias else None
    layers = _row_layers(qW, qs, world, bias, True)
    full = _row_full(layers, x)
    Ss = x.shape[0] // world
    for route in ("stage", "fused"):
        outs = _row_sp(layers, x, route)
        torch.cuda.synchronize()
        nat.check()
        for r in range(world):
            assert torch.equal(outs[r], full[r * Ss:(r + 1) * Ss]), f"{route}, rank {r}"


@pytest.mark.parametrize("M", [1, 4, 16, 256, 4096])
@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32", "tf32"])
@pytest.mark.parametrize("nested,with_bias", [(False, False), (True, True)])
def test_one_rank_sp_is_matmul_4bit(precision, M, dtype, nested, with_bias):
    import bitsandbytes_b200 as bnb
    from bitsandbytes_b200.parallel import RowParallelLinear4bit

    precision("tf32" if dtype == "tf32" else "ieee")
    td = _DT[dtype]
    N, K = 1280, 1024
    qW, qs = _quantized(N, K, td, nested, M, "fp4")
    g = torch.Generator().manual_seed(M)
    x = torch.randn(M, K, generator=g).to(td).cuda()
    bias = torch.randn(N, generator=g).to(td).cuda() if with_bias else None
    layer = RowParallelLinear4bit.from_quantized(qW, qs, bias=bias, sequence_parallel=True)
    got = layer(x)
    want = bnb.matmul_4bit(x, qW.t(), qs, bias=bias)
    torch.cuda.synchronize()
    assert got.shape == (M, N) and torch.equal(got, want)


def _col_layers(qW, qs, world, bias, sp):
    from bitsandbytes_b200.parallel import ColumnParallelLinear4bit, slice_quantized_weight

    return [ColumnParallelLinear4bit(slice_quantized_weight(qW, qs, world, r), qs.shape[0], bias, gather_output=False,
                                     sequence_parallel=sp) for r in range(world)]


def _col_sp(layers, x, route):
    """Every rank's SP column output from the ranks' token shards.  stage: one gathered [M, K] copy (what the
    all-gather produces).  fused: each rank copies its shard into its rows of every rank's own [M, K] buffer."""
    world = len(layers)
    Ms = x.shape[0] // world
    shards = [x[r * Ms:(r + 1) * Ms].clone() for r in range(world)]
    if route == "stage":
        gathered = [torch.cat(shards)] * world
    else:
        gathered = [torch.full_like(x, float("nan")) for _ in range(world)]
        for r in range(world):
            for s in range(world):
                gathered[s][r * Ms:(r + 1) * Ms].copy_(shards[r])
    return [L.local_forward(gathered[r]).view(*x.shape[:-1], L.shard.rows) for r, L in enumerate(layers)]


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("M", [8, 256, 4096])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_column_layer_sp_is_the_non_sp_output(world, M, dtype):
    N, K = 2048, 1024
    qW, qs = _quantized(N, K, dtype, False, M + world)
    g = torch.Generator().manual_seed(world)
    x = torch.randn(M, K, generator=g).to(dtype).cuda()
    bias = torch.randn(N, generator=g).to(dtype).cuda()
    sp, plain = _col_layers(qW, qs, world, bias, True), _col_layers(qW, qs, world, bias, False)
    for route in ("stage", "fused"):
        outs = _col_sp(sp, x, route)
        torch.cuda.synchronize()
        for r in range(world):
            assert torch.equal(outs[r], plain[r](x)), f"{route}, rank {r}"


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("M", [16, 256])
def test_sp_mlp_chain(world, M):
    """column(SP) -> SiLU -> row(SP) gives the token slices of column(gather_output=False) -> SiLU -> row."""
    dt = torch.bfloat16
    H, I = 1024, 2048
    up_q, up_s = _quantized(I, H, dt, False, 1)
    down_q, down_s = _quantized(H, I, dt, True, 2)
    g = torch.Generator().manual_seed(M)
    x = torch.randn(M, H, generator=g).to(dt).cuda()
    b_up, b_down = (torch.randn(n, generator=g).to(dt).cuda() for n in (I, H))
    up_sp, up = _col_layers(up_q, up_s, world, b_up, True), _col_layers(up_q, up_s, world, b_up, False)
    down_sp, down = _row_layers(down_q, down_s, world, b_down, True), _row_layers(down_q, down_s, world, b_down, False)
    h = [torch.nn.functional.silu(L(x)) for L in up]
    full = _row_full_sharded(down, h)
    for route in ("stage", "fused"):
        h_sp = [torch.nn.functional.silu(y) for y in _col_sp(up_sp, x, route)]
        y_sp = _row_sp_sharded(down_sp, h_sp, route)
        torch.cuda.synchronize()
        Ms = M // world
        for r in range(world):
            assert torch.equal(y_sp[r], full[r * Ms:(r + 1) * Ms]), f"{route}, rank {r}"


def _row_full_sharded(layers, hs):
    from bitsandbytes_b200.backends.cuda import reduce_partials

    M, N = hs[0].shape[0], layers[0].out_features
    stage = torch.empty((len(layers), M, N), device="cuda")
    for r, L in enumerate(layers):
        assert L.partial_forward(hs[r], [stage[r]])
    return reduce_partials(stage, hs[0].dtype, layers[0].bias)


def _row_sp_sharded(layers, hs, route):
    """_row_sp with each rank's own input slice (the column layer's output) instead of a slice of one x."""
    from bitsandbytes_b200.backends.cuda import reduce_partials

    world = len(layers)
    M, N = hs[0].shape[0], layers[0].out_features
    Ms = M // world
    bufs = [torch.full((world, Ms, N), float("nan"), device="cuda") for _ in range(world)]
    for r, L in enumerate(layers):
        if route == "stage":
            send = torch.empty((world, Ms, N), device="cuda")
            assert L.partial_forward(hs[r], [send])
            for s in range(world):
                bufs[s][r].copy_(send[s])
        else:
            assert L.partial_scatter(hs[r], [b.data_ptr() + r * Ms * N * 4 for b in bufs])
    return [reduce_partials(bufs[r], hs[0].dtype, L.bias) for r, L in enumerate(layers)]


def test_fused_sp_routes_replay_in_a_cuda_graph():
    """The fused column (shard copies) and row (scatter GEMM) routes of four ranks plus the reductions, captured once
    and replayed on three new inputs: the eager bits."""
    dt = torch.bfloat16
    world, M, H, I = 4, 64, 1024, 2048
    up_q, up_s = _quantized(I, H, dt, False, 3)
    down_q, down_s = _quantized(H, I, dt, False, 4)
    up = _col_layers(up_q, up_s, world, None, True)
    down = _row_layers(down_q, down_s, world, torch.randn(H).to(dt).cuda(), True)

    def step(x):
        return _row_sp_sharded(down, _col_sp(up, x, "fused"), "fused")

    static_x = torch.randn(M, H).to(dt).cuda()
    step(static_x)  # warm-up: module loads, workspace
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step(static_x)
    for seed in range(3):
        static_x.copy_(torch.randn(M, H, generator=torch.Generator().manual_seed(seed)).to(dt).cuda())
        graph.replay()
        eager = step(static_x)
        torch.cuda.synchronize()
        for a, b in zip(outs, eager):
            assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------ processes
_SCRIPT = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import bitsandbytes_b200.functional as F
from bitsandbytes_b200.parallel import (ColumnParallelLinear4bit, PeerGather, PeerPartials, RowParallelLinear4bit,
                                        fused_forward_col_sp, fused_forward_row_sp)
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
H, I = 2048, 4096
for M in (8, 48, 1024):
    torch.manual_seed(0)
    up_q, up_s = F.quantize_4bit((torch.randn(I, H, device=dev) / H**0.5).to(torch.bfloat16), quant_type="nf4")
    dn_q, dn_s = F.quantize_4bit((torch.randn(H, I, device=dev) / I**0.5).to(torch.bfloat16), quant_type="fp4",
                                 compress_statistics=True)
    x = torch.randn(M, H, device=dev, dtype=torch.bfloat16)
    b = torch.randn(H, device=dev, dtype=torch.bfloat16)
    Ms = M // world
    xs = x[rank * Ms:(rank + 1) * Ms].contiguous()
    up = ColumnParallelLinear4bit.from_quantized(up_q, up_s, gather_output=False)
    dn = RowParallelLinear4bit.from_quantized(dn_q, dn_s, bias=b)
    up_sp = ColumnParallelLinear4bit.from_quantized(up_q, up_s, gather_output=False, sequence_parallel=True)
    dn_sp = RowParallelLinear4bit.from_quantized(dn_q, dn_s, bias=b, sequence_parallel=True)
    want = dn(torch.nn.functional.silu(up(x)))[rank * Ms:(rank + 1) * Ms]
    h = up_sp(xs)
    assert torch.equal(h, up(x)), f"M={M}: SP column differs"
    nccl = dn_sp(torch.nn.functional.silu(h))
    gather, parts = PeerGather(M, H, torch.bfloat16, dev), PeerPartials(Ms, H, dev)
    fused = []
    for _ in range(3):
        hf = fused_forward_col_sp(up_sp, xs, gather)
        fused.append(fused_forward_row_sp(dn_sp, torch.nn.functional.silu(hf), parts).clone())
    torch.cuda.synchronize()
    assert torch.equal(nccl, want), f"M={M}: SP row (NCCL) differs from the non-SP rows"
    assert all(torch.equal(f, nccl) for f in fused), f"M={M}: fused SP differs from NCCL SP"
dist.barrier()
dist.destroy_process_group()
print("SP_OK", rank)
"""


@pytest.mark.parametrize("nproc", [1, 2])
def test_processes_fused_equals_nccl(tmp_path, nproc):
    """One process per GPU: the SP MLP through symmetric memory and through NCCL give the non-SP rows bit for bit on
    every rank.  One process exercises the symmetric-memory routes; two need two GPUs."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "sp.py"
    script.write_text(_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29581 + nproc), str(script)],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and r.stdout.count("SP_OK") == nproc, r.stdout[-2000:] + r.stderr[-3000:]
