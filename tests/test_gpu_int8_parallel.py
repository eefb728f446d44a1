"""GPU tests of the tensor-parallel LLM.int8() layers on one H100: worlds of 1, 2, 4 and 8 simulated rank by rank, for
the column- and the row-parallel layer and both exchange routes (a staging buffer as NCCL fills it, and the GEMM's
stores into every rank's buffer).  Every rank's output must equal the unsharded inference Linear8bitLt output bit for
bit, with and without outlier columns, up to and past the 64 columns the fused epilogue takes."""
import os
import subprocess
import sys

import pytest
import torch

from tests import _native as nat

pytestmark = pytest.mark.gpu

_DT = {"fp16": torch.float16, "bf16": torch.bfloat16}
N_, K_ = 512, 1024  # K / 8 = 128: every world up to 8 keeps its shard on the int8 GEMM


def _reference(M, dtype, with_bias, threshold, cols=(), seed=0, N=N_, K=K_):
    """(x, the unsharded Linear8bitLt, its output, CB, SCB, bias) with outlier entries injected into ``cols``."""
    import bitsandbytes_b200 as bnb
    from bitsandbytes_b200.parallel import _state_of

    g = torch.Generator().manual_seed(seed)
    lin = bnb.nn.Linear8bitLt(K, N, bias=with_bias, has_fp16_weights=False, threshold=threshold)
    with torch.no_grad():
        lin.weight.data = (torch.randn(N, K, generator=g) / K**0.5).to(torch.float16)
        if with_bias:
            lin.bias.data = torch.randn(N, generator=g).to(torch.float16)
    lin = lin.cuda().eval()
    x = torch.randn(M, K, generator=g) * 0.5
    for i, c in enumerate(cols):
        x[i % M::3, c] = 7.0 + (i % 5) if i % 2 == 0 else -7.5
    x = x.to(dtype).cuda()
    with torch.no_grad():
        y = lin(x)
    CB, SCB, _ = _state_of(lin)
    bias = lin.bias.data if with_bias else None
    return x, lin, y, CB, SCB, bias


def _col_layers(CB, SCB, bias, world, threshold):
    from bitsandbytes_b200.parallel import ColumnParallelLinear8bitLt, slice_int8_weight

    return [ColumnParallelLinear8bitLt(slice_int8_weight(CB, SCB, world, r), CB.shape[0], bias, threshold=threshold)
            for r in range(world)]


def _row_layers(CB, SCB, bias, world, threshold):
    from bitsandbytes_b200.parallel import RowParallelLinear8bitLt, slice_int8_weight_k

    return [RowParallelLinear8bitLt(slice_int8_weight_k(CB, SCB, world, r), CB.shape[1], bias, input_is_parallel=False,
                                    threshold=threshold) for r in range(world)]


def _simulate_col(layers, x, route):
    """Every rank's [M, N] output.  stage: each rank's columns into its slot of a [w, M, N/w] stage, gathered.  fused:
    each rank's GEMM stores its columns into every rank's [M, N] buffer (past 64 outlier columns: the stage route)."""
    world = len(layers)
    N, rows = layers[0].out_features, layers[0].shard.rows
    qs = [L.quantize(x) for L in layers]
    M = qs[0].A.shape[0]
    J = qs[0].J
    if route == "fused" and J <= 64:
        bufs = [torch.full((M, N), float("nan"), device="cuda", dtype=x.dtype) for _ in range(world)]
        for L, q in zip(layers, qs):
            col = L.shard.row0 * x.element_size()
            assert L._gemm(q, [b.data_ptr() + col for b in bufs], N)
        return bufs
    stage = torch.full((world, M, rows), float("nan"), device="cuda", dtype=x.dtype)
    for r, (L, q) in enumerate(zip(layers, qs)):
        L.local_forward(q, stage[r], rows)
    full = stage.permute(1, 0, 2).reshape(M, N)
    if J > 64:
        subBT = torch.cat([L.outlier_rows(q) for L, q in zip(layers, qs)])
        full = layers[0].finish(full, qs[0], subBT)
    return [full] * world


def _simulate_row(layers, x, route):
    """Every rank's [M, N] output: local statistics, their max over the ranks, codes, int32 partials (into one shared
    stage, or stored by each GEMM into slot r of every rank's buffer), the outlier operands in rank order, reduction."""
    world = len(layers)
    xs = [L.local_input(x) for L in layers]
    sts = [L.local_stats(xr) for L, xr in zip(layers, xs)]
    SCA = torch.stack([st.row_stats for st in sts]).amax(0)
    codes = [L.local_codes(st, SCA) for L, st in zip(layers, sts)]
    M, N = xs[0].shape[0], layers[0].out_features
    if route == "stage":
        stage = torch.full((world, M, N), -1, device="cuda", dtype=torch.int32)
        for r, (L, (CA, _)) in enumerate(zip(layers, codes)):
            assert L.partial_forward(CA, [stage[r]])
        parts = [stage] * world
    else:
        parts = [torch.full((world, M, N), -1, device="cuda", dtype=torch.int32) for _ in range(world)]
        for r, (L, (CA, _)) in enumerate(zip(layers, codes)):
            assert L.partial_forward(CA, [p.data_ptr() + r * M * N * 4 for p in parts])
    subA = subBT = None
    if codes[0][1] is not None:
        counts = [int(c.numel()) for _, c in codes]
        if sum(counts):
            P = max(8, -(-max(counts) // 8) * 8)
            ops = [L.outlier_operands(xr, c, P) for L, xr, (_, c) in zip(layers, xs, codes)]
            subA, subBT = layers[0].combine_outliers(ops, counts)
    return [L.reduce(p, SCA, x.dtype, subA, subBT) for L, p in zip(layers, parts)]


def _check_all(x, y, CB, SCB, bias, world, threshold):
    for kind, make, sim in (("col", _col_layers, _simulate_col), ("row", _row_layers, _simulate_row)):
        layers = make(CB, SCB, bias, world, threshold)
        for route in ("stage", "fused"):
            outs = sim(layers, x, route)
            torch.cuda.synchronize()
            nat.check()
            for r, o in enumerate(outs):
                assert o.shape == y.shape
                same = o.view(torch.int16) == y.view(torch.int16)
                assert bool(same.all()), f"{kind}/{route} rank {r}: {int((~same).sum())} / {same.numel()} differ"


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("M", [1, 2, 16, 256, 4096])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("with_bias", [False, True])
def test_threshold_zero_equals_linear8bitlt(world, M, dtype, with_bias):
    x, _, y, CB, SCB, bias = _reference(M, _DT[dtype], with_bias, 0.0, seed=M + world)
    _check_all(x, y, CB, SCB, bias, world, 0.0)


def _outlier_cols(J, placement, K=K_):
    if placement == "one_shard":  # all inside [128, 256): one shard at world 8, inside one at every smaller world too
        return [128 + i for i in range(J)]
    # spread over K, with columns on both sides of every 1/8 boundary
    edges = [b + d for b in range(K // 8, K, K // 8) for d in (-1, 0)]
    rest = [c for c in range(3, K, max(1, K // max(J, 1)) | 1) if c not in edges]
    return sorted((edges + rest)[:J])


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("J", [1, 5, 41, 64, 65, 100])
@pytest.mark.parametrize("placement", ["spread", "one_shard"])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_outlier_columns_equal_linear8bitlt(world, J, placement, dtype):
    cols = _outlier_cols(J, placement)
    assert len(set(cols)) == J
    x, lin, y, CB, SCB, bias = _reference(16, _DT[dtype], True, 6.0, cols, seed=J + world)
    assert int(lin.state.idx.numel()) == J  # the unsharded layer sees exactly these outlier columns
    _check_all(x, y, CB, SCB, bias, world, 6.0)


@pytest.mark.parametrize("M", [1, 2, 256, 4096])
@pytest.mark.parametrize("J", [5, 65])
@pytest.mark.parametrize("with_bias", [False, True])
def test_outlier_columns_every_m(M, J, with_bias):
    x, _, y, CB, SCB, bias = _reference(M, torch.bfloat16, with_bias, 6.0, _outlier_cols(J, "spread"), seed=M)
    _check_all(x, y, CB, SCB, bias, 4, 6.0)


@pytest.mark.parametrize("kind", ["col", "row"])
@pytest.mark.parametrize("threshold", [0.0, 6.0])
def test_module_forward_one_rank(kind, threshold):
    """forward() of a one-rank layer built from the module: the unsharded output, including a 3-D input."""
    from bitsandbytes_b200.parallel import ColumnParallelLinear8bitLt, RowParallelLinear8bitLt

    x, lin, y, _, _, _ = _reference(48, torch.float16, True, threshold, _outlier_cols(70, "spread") if threshold else (),
                                    seed=7)
    cls = ColumnParallelLinear8bitLt if kind == "col" else RowParallelLinear8bitLt
    layer = cls.from_linear8bitlt(lin)
    got = layer(x.view(2, 24, K_))
    assert got.shape == (2, 24, N_)
    assert torch.equal(got.view(48, N_), y)


def test_quant_halves_equal_the_one_pass_quantiser():
    """Statistics-only and codes-from-statistics give exactly the one-pass kernel's statistics, flags and codes."""
    from bitsandbytes_b200.backends.cuda import int8_quant_with_stats, int8_row_stats, int8_vectorwise_quant_flags

    for dtype in (torch.float16, torch.bfloat16):
        for cols in (1024, 1000, 9000):
            g = torch.Generator().manual_seed(cols)
            A = (torch.randn(33, cols, generator=g) * 3).to(dtype).cuda()
            for thr in (0.0, 6.0):
                q, stats, flags = int8_vectorwise_quant_flags(A, thr)
                s2, f2 = int8_row_stats(A, thr)
                q2 = int8_quant_with_stats(A, s2, thr)
                torch.cuda.synchronize()
                assert torch.equal(s2.view(torch.int32), stats.view(torch.int32))
                assert (f2 is None) == (flags is None) and (flags is None or torch.equal(f2, flags))
                assert torch.equal(q2, q)


@pytest.mark.parametrize("M", [1, 5, 128, 300])
@pytest.mark.parametrize("form", ["int32", "fp16", "bf16", "bf16_outliers"])
def test_eight_destinations_hold_the_one_destination_bits(M, form):
    """n_outs = 8 local buffers standing in for peers at a ragged row stride: each holds the bits of n_outs = 1, which
    are those of the library's single-GPU ops, and nothing outside [M, N] is written."""
    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.backends.cuda import int8_gemm_multi_out, int8_outlier_operands

    N, K = 1000, 512
    ldc = N + 3
    g = torch.Generator().manual_seed(M)
    A = torch.randn(M, K, generator=g).half().cuda()
    W = torch.randn(N, K, generator=g).half().cuda()
    CA, SCA, _ = F.int8_vectorwise_quant(A)
    CB, SCB, _ = F.int8_vectorwise_quant(W)
    dtype = None if form == "int32" else _DT[form[:4]]
    bias = None if dtype is None else torch.randn(N, generator=g).to(dtype).cuda()
    subA = subBT = None
    cols = torch.tensor([3, 17, 100, 511, 200], device="cuda")
    if form == "bf16_outliers":
        subA, subBT = int8_outlier_operands(A.to(dtype), CB, SCB, cols)
    out_dt = torch.int32 if dtype is None else dtype

    def run(n):
        outs = [torch.full((M, ldc), -7, device="cuda", dtype=out_dt) for _ in range(n)]
        assert int8_gemm_multi_out(CA, CB, SCA, SCB, outs, ldc, dtype, bias, subA, subBT)
        return outs

    one, eight = run(1)[0], run(8)
    torch.cuda.synchronize()
    nat.check()
    assert (one[:, N:] == -7).all()
    for o in eight:
        assert torch.equal(o, one)
    if dtype is None:
        want = torch.ops.bitsandbytes.int8_linear_matmul.default(CA, CB)
    elif subA is None:
        want = torch.ops.bitsandbytes.int8_scaled_mm.default(CA, CB, SCA, SCB, bias=bias, dtype=dtype)
    else:
        want, _ = torch.ops.bitsandbytes.int8_mixed_scaled_mm(A.to(dtype), CA, CB, SCA, SCB, cols, bias)
    assert torch.equal(one[:, :N], want)


def test_threshold_zero_fused_routes_replay_in_a_cuda_graph():
    """Both layers' fused routes for a world of 4 simulated rank by rank, captured once and replayed on new inputs:
    the eager bits, which are the unsharded layer's."""
    x, _, _, CB, SCB, bias = _reference(64, torch.bfloat16, True, 0.0, seed=11)
    cols, rows = _col_layers(CB, SCB, bias, 4, 0.0), _row_layers(CB, SCB, bias, 4, 0.0)
    static_x = x.clone()

    def step():
        return _simulate_col(cols, static_x, "fused") + _simulate_row(rows, static_x, "fused")

    step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for seed in range(3):
        xn = (torch.randn(64, K_, generator=torch.Generator().manual_seed(100 + seed)) * 0.5).to(torch.bfloat16).cuda()
        static_x.copy_(xn)
        graph.replay()
        eager = step()
        torch.cuda.synchronize()
        for a, b in zip(outs, eager):
            assert torch.equal(a, b)


@pytest.mark.parametrize("kind", ["col", "row"])
def test_capture_with_threshold_raises(kind):
    x, lin, _, CB, SCB, bias = _reference(16, torch.float16, False, 6.0, seed=2)
    layer = (_col_layers if kind == "col" else _row_layers)(CB, SCB, bias, 1, 6.0)[0]
    layer(x)  # eager is fine
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="capture"):
        with torch.cuda.graph(graph):
            layer(x)


def test_wrapper_checks():
    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.backends.cuda import int8_gemm_multi_out, int8_reduce_partials

    CA, SCA, _ = F.int8_vectorwise_quant(torch.randn(8, 64, device="cuda").half())
    CB, SCB, _ = F.int8_vectorwise_quant(torch.randn(32, 64, device="cuda").half())
    with pytest.raises(ValueError):
        int8_gemm_multi_out(CA, CB, SCA, SCB, [torch.empty(8, 32, device="cuda")], 32, torch.float16)  # not fp16
    with pytest.raises(ValueError):
        int8_gemm_multi_out(CA, CB, None, None, [torch.empty(8, 32, device="cuda", dtype=torch.int32)] * 9, 32, None)
    with pytest.raises(ValueError):
        int8_gemm_multi_out(CA, CB, None, None, [torch.empty(8 * 32 - 1, device="cuda", dtype=torch.int32)], 32, None)
    with pytest.raises(ValueError):
        int8_reduce_partials(torch.zeros(2, 8, 32, device="cuda"), SCA, SCB, torch.float16)  # not int32
    with pytest.raises(ValueError):
        int8_reduce_partials(torch.zeros(2, 8, 32, device="cuda", dtype=torch.int32), SCA, SCB[:7], torch.float16)


# ------------------------------------------------------------------------------------------ processes
_SCRIPT = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import bitsandbytes_b200 as bnb
from bitsandbytes_b200.parallel import (ColumnParallelLinear8bitLt, PeerGather, PeerPartials, RowParallelLinear8bitLt,
                                        fused_forward_col8, fused_forward_row8)
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
N, K = 1024, 2048
for M, thr, J in ((1, 0.0, 0), (48, 6.0, 5), (256, 6.0, 80)):
    torch.manual_seed(0)
    lin = bnb.nn.Linear8bitLt(K, N, bias=True, has_fp16_weights=False, threshold=thr)
    lin.weight.data = (torch.randn(N, K) / K**0.5).half()
    lin = lin.to(dev).eval()
    x = (torch.randn(M, K, device=dev) * 0.5).to(torch.bfloat16)
    x[:, torch.arange(J, device=dev) * (K // max(J, 1))] = 7.0
    with torch.no_grad():
        single = lin(x)
    col = ColumnParallelLinear8bitLt.from_linear8bitlt(lin)
    row = RowParallelLinear8bitLt.from_linear8bitlt(lin, input_is_parallel=False)
    gather, parts = PeerGather(M, N, torch.bfloat16, dev), PeerPartials(M, N, dev, dtype=torch.int32)
    for name, nccl, fused in (("col", col(x), [fused_forward_col8(col, x, gather).clone() for _ in range(3)]),
                              ("row", row(x), [fused_forward_row8(row, x, parts).clone() for _ in range(3)])):
        torch.cuda.synchronize()
        assert torch.equal(nccl, single), f"{name} M={M}: NCCL route differs from Linear8bitLt"
        assert all(torch.equal(f, nccl) for f in fused), f"{name} M={M}: fused route differs from the NCCL one"
dist.barrier()
dist.destroy_process_group()
print("INT8_TP_OK", rank)
"""


@pytest.mark.parametrize("nproc", [1, 2])
def test_processes_fused_equals_nccl(tmp_path, nproc):
    """One process per GPU: the symmetric-memory and the NCCL exchanges give the unsharded bits on every rank.  Two
    processes need two GPUs."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "int8_tp.py"
    script.write_text(_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29571 + nproc), str(script)],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and r.stdout.count("INT8_TP_OK") == nproc, r.stdout[-2000:] + r.stderr[-3000:]
