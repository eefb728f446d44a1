"""GPU tests of the sequence-parallel LLM.int8() layers on one H100: the int32 scatter GEMM against the broadcast one,
worlds of 2, 4 and 8 simulated rank by rank for the row and column layers (both exchange routes, threshold 0 and up to
and past the 64 outlier columns the fused epilogue takes) and a column -> GELU -> row chain, world 1 against
Linear8bitLt, a CUDA-graph replay of the fused routes, and the one- / two-process runs.  Every output must be the
unsharded Linear8bitLt's bits: the row layer's the rows of the rank's tokens, the column layer's its feature columns."""
import os
import subprocess
import sys

import pytest
import torch

from tests import _native as nat
from tests.test_gpu_int8_parallel import K_, N_, _outlier_cols, _reference

pytestmark = pytest.mark.gpu

_DT = {"fp16": torch.float16, "bf16": torch.bfloat16}


@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("Ms", [1, 5, 32, 128, 300])
def test_scatter_equals_broadcast(world, Ms):
    """Rank s's rows of the one-destination int32 partial land in destination s, and every other byte keeps the
    sentinel: columns past N at a ragged row stride, and the row after each destination's share.  At Ms < 128 one
    128-token tile spans up to 8 destinations."""
    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.backends.cuda import int8_gemm_multi_out, int8_gemm_partial_scatter

    M, N, K = world * Ms, 1000, 512
    ldc = N + 3
    g = torch.Generator().manual_seed(world * 1000 + Ms)
    CA, _, _ = F.int8_vectorwise_quant(torch.randn(M, K, generator=g).half().cuda())
    CB, _, _ = F.int8_vectorwise_quant(torch.randn(N, K, generator=g).half().cuda())
    sentinel = -123456789
    one = torch.full((M, ldc), sentinel, device="cuda", dtype=torch.int32)
    assert int8_gemm_multi_out(CA, CB, None, None, [one], ldc, None)
    outs = [torch.full((Ms + 1, ldc), sentinel, device="cuda", dtype=torch.int32) for _ in range(world)]
    assert int8_gemm_partial_scatter(CA, CB, [o[:Ms] for o in outs], ldc)
    torch.cuda.synchronize()
    nat.check()
    assert torch.equal(one[:, :N], torch.ops.bitsandbytes.int8_linear_matmul.default(CA, CB))
    for s, o in enumerate(outs):
        assert torch.equal(o[:Ms], one[s * Ms:(s + 1) * Ms]), f"destination {s}"
        assert (o[:, N:] == sentinel).all() and (o[Ms] == sentinel).all(), f"destination {s}: stray store"


# ------------------------------------------------------------------------------------------ row layer
def _row_layers(CB, SCB, bias, world, threshold, input_is_parallel=False):
    from bitsandbytes_b200.parallel import RowParallelLinear8bitLt, slice_int8_weight_k

    return [RowParallelLinear8bitLt(slice_int8_weight_k(CB, SCB, world, r), CB.shape[1], bias,
                                    input_is_parallel=input_is_parallel, threshold=threshold, sequence_parallel=True)
            for r in range(world)]


def _row_sp(layers, inputs, route):
    """Every rank's SP output [M/w, N], the ranks run in turn through the layer's steps: local statistics, their max,
    codes, the outlier counts; up to 64 outlier columns the partials of rank s's tokens reach rank s (stage: each
    rank's full partial, chunk s copied to rank s, as the all-to-all does; fused: the scatter GEMM into slot r of every
    rank's buffer) and each rank reduces them with its rows of SCA and subA; past 64 the non-SP result's rows."""
    world = len(layers)
    xs = [L.local_input(x) for L, x in zip(layers, inputs)]
    dtype = inputs[0].dtype
    sts = [L.local_stats(xr) for L, xr in zip(layers, xs)]
    SCA = torch.stack([st.row_stats for st in sts]).amax(0)
    codes = [L.local_codes(st, SCA) for L, st in zip(layers, sts)]
    M, N = xs[0].shape[0], layers[0].out_features
    Ms = M // world
    subA = subBT = None
    J = 0
    if codes[0][1] is not None:
        counts = [int(c.numel()) for _, c in codes]
        J = sum(counts)
        if J:
            P = max(8, -(-max(counts) // 8) * 8)
            ops = [L.outlier_operands(xr, c, P) for L, xr, (_, c) in zip(layers, xs, codes)]
            subA, subBT = layers[0].combine_outliers(ops, counts)
    if J > 64:
        stage = torch.full((world, M, N), -1, device="cuda", dtype=torch.int32)
        for r, (L, (CA, _)) in enumerate(zip(layers, codes)):
            assert L.partial_forward(CA, [stage[r]])
        full = layers[0].reduce(stage, SCA, dtype, subA, subBT)
        return [full[r * Ms:(r + 1) * Ms] for r in range(world)]
    bufs = [torch.full((world, Ms, N), -1, device="cuda", dtype=torch.int32) for _ in range(world)]
    for r, (L, (CA, _)) in enumerate(zip(layers, codes)):
        if route == "stage":
            send = torch.full((world, Ms, N), -1, device="cuda", dtype=torch.int32)
            assert L.partial_forward(CA, [send])
            for s in range(world):
                bufs[s][r].copy_(send[s])
        else:
            assert L.partial_scatter(CA, [b.data_ptr() + r * Ms * N * 4 for b in bufs])
    outs = []
    for r, L in enumerate(layers):
        rows = slice(r * Ms, (r + 1) * Ms)
        outs.append(L.reduce(bufs[r], SCA[rows], dtype, None if subA is None else subA[rows], subBT))
    return outs


def _check_row(x, y, CB, SCB, bias, world, threshold):
    layers = _row_layers(CB, SCB, bias, world, threshold)
    Ms = x.shape[0] // world
    for route in ("stage", "fused"):
        outs = _row_sp(layers, [x] * world, route)
        torch.cuda.synchronize()
        nat.check()
        for r, o in enumerate(outs):
            want = y[r * Ms:(r + 1) * Ms]
            same = o.view(torch.int16) == want.view(torch.int16)
            assert o.shape == want.shape and bool(same.all()), f"row/{route} rank {r}: {int((~same).sum())} differ"


_WM = [(w, M) for w in (2, 4, 8) for M in (w, 16, 256, 4096)]


@pytest.mark.parametrize("world,M", _WM)
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("with_bias", [False, True])
def test_row_layer_threshold_zero(world, M, dtype, with_bias):
    x, _, y, CB, SCB, bias = _reference(M, _DT[dtype], with_bias, 0.0, seed=M + world)
    _check_row(x, y, CB, SCB, bias, world, 0.0)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("J", [0, 1, 5, 41, 64, 65, 100])
@pytest.mark.parametrize("placement", ["spread", "one_shard"])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_row_layer_outlier_columns(world, J, placement, dtype):
    x, lin, y, CB, SCB, bias = _reference(16, _DT[dtype], True, 6.0, _outlier_cols(J, placement), seed=J + world)
    assert int(lin.state.idx.numel()) == J
    _check_row(x, y, CB, SCB, bias, world, 6.0)


@pytest.mark.parametrize("world,M", _WM)
@pytest.mark.parametrize("J", [5, 65])
@pytest.mark.parametrize("with_bias", [False, True])
def test_row_layer_outliers_every_m(world, M, J, with_bias):
    x, _, y, CB, SCB, bias = _reference(M, torch.float16, with_bias, 6.0, _outlier_cols(J, "spread"), seed=M + J)
    _check_row(x, y, CB, SCB, bias, world, 6.0)


# ------------------------------------------------------------------------------------------ column layer
def _col_layers(CB, SCB, bias, world, threshold):
    from bitsandbytes_b200.parallel import ColumnParallelLinear8bitLt, slice_int8_weight

    return [ColumnParallelLinear8bitLt(slice_int8_weight(CB, SCB, world, r), CB.shape[0], bias, gather_output=False,
                                       threshold=threshold, sequence_parallel=True) for r in range(world)]


def _col_sp(layers, x, route):
    """Every rank's SP column output [M, N/w] from the ranks' token shards, through the layer's steps: local
    quantisation, the union of the flags, the zeroing and the local outlier operands, the gathered codes, statistics
    and outlier columns (stage: one concatenated copy, as the all-gather produces; fused: each rank copies its rows into
    every rank's own buffer), then the GEMM; past 64 outlier columns the gathered output and the addmm."""
    from bitsandbytes_b200.parallel import Int8Input

    world = len(layers)
    M, K = x.shape[0], x.shape[-1]
    Ms = M // world
    loc = [L.local_quantize(x[r * Ms:(r + 1) * Ms]) for r, L in enumerate(layers)]
    cols = None
    if loc[0][3] is not None:
        cols = torch.nonzero(torch.stack([f for *_, f in loc]).amax(0)).view(-1)
    ops = [L.local_outliers(xs, CA, cols, M) for L, (xs, CA, _, _) in zip(layers, loc)]
    if route == "stage":
        CAs = [torch.cat([CA for _, CA, _, _ in loc])] * world
        SCAs = [torch.cat([SCA for _, _, SCA, _ in loc])] * world
    else:
        CAs = [torch.full((M, K), 77, device="cuda", dtype=torch.int8) for _ in range(world)]
        SCAs = [torch.full((M,), float("nan"), device="cuda") for _ in range(world)]
        for r, (_, CA, SCA, _) in enumerate(loc):
            for s in range(world):
                CAs[s][r * Ms:(r + 1) * Ms].copy_(CA)
                SCAs[s][r * Ms:(r + 1) * Ms].copy_(SCA)
    subA = None if ops[0][0] is None else torch.cat([a for a, _ in ops])
    qs = [Int8Input(None, CAs[r], SCAs[r], cols, x.dtype, subA, ops[r][1]) for r in range(world)]
    if qs[0].J <= 64:
        return [L.local_forward(q) for L, q in zip(layers, qs)]
    full = torch.cat([L.local_forward(q) for L, q in zip(layers, qs)], dim=1)
    full = layers[0].finish(full, qs[0], torch.cat([L.outlier_rows(q) for L, q in zip(layers, qs)]))
    return [full[:, L.shard.row0:L.shard.row0 + L.shard.rows] for L in layers]


def _check_col(x, y, CB, SCB, bias, world, threshold):
    from tests.test_gpu_int8_parallel import _col_layers as plain_layers, _simulate_col

    plain = _simulate_col(plain_layers(CB, SCB, bias, world, threshold), x, "stage")[0]  # the non-SP layer
    assert torch.equal(plain, y)
    layers = _col_layers(CB, SCB, bias, world, threshold)
    for route in ("stage", "fused"):
        outs = _col_sp(layers, x, route)
        torch.cuda.synchronize()
        nat.check()
        for r, (L, o) in enumerate(zip(layers, outs)):
            want = plain[:, L.shard.row0:L.shard.row0 + L.shard.rows]
            same = o.view(torch.int16) == want.view(torch.int16)
            assert o.shape == want.shape and bool(same.all()), f"col/{route} rank {r}: {int((~same).sum())} differ"


@pytest.mark.parametrize("world,M", _WM)
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("with_bias", [False, True])
def test_column_layer_threshold_zero(world, M, dtype, with_bias):
    x, _, y, CB, SCB, bias = _reference(M, _DT[dtype], with_bias, 0.0, seed=M + world)
    _check_col(x, y, CB, SCB, bias, world, 0.0)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("J", [0, 1, 5, 41, 64, 65, 100])
@pytest.mark.parametrize("placement", ["spread", "one_shard"])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_column_layer_outlier_columns(world, J, placement, dtype):
    x, lin, y, CB, SCB, bias = _reference(16, _DT[dtype], True, 6.0, _outlier_cols(J, placement), seed=J + world)
    assert int(lin.state.idx.numel()) == J
    _check_col(x, y, CB, SCB, bias, world, 6.0)


@pytest.mark.parametrize("world,M", _WM)
@pytest.mark.parametrize("J", [5, 65])
def test_column_layer_outliers_every_m(world, M, J):
    x, _, y, CB, SCB, bias = _reference(M, torch.bfloat16, True, 6.0, _outlier_cols(J, "spread"), seed=M + J)
    _check_col(x, y, CB, SCB, bias, world, 6.0)


@pytest.mark.parametrize("world,M", [(2, 16), (8, 64), (8, 8)])
def test_column_outliers_in_one_rank_only(world, M):
    """Outlier entries only in rank 0's tokens: every other rank must still zero those columns in its codes.  With
    (8, 8) each rank holds a single token, and the columns are zeroed all the same (the global M is what counts)."""
    import bitsandbytes_b200 as bnb
    from bitsandbytes_b200.parallel import _state_of

    g = torch.Generator().manual_seed(M)
    lin = bnb.nn.Linear8bitLt(K_, N_, bias=True, has_fp16_weights=False, threshold=6.0)
    with torch.no_grad():
        lin.weight.data = (torch.randn(N_, K_, generator=g) / K_**0.5).to(torch.float16)
        lin.bias.data = torch.randn(N_, generator=g).to(torch.float16)
    lin = lin.cuda().eval()
    x = torch.randn(M, K_, generator=g) * 0.5
    x[0, [3, 200, 777]] = torch.tensor([8.0, -9.0, 7.5])  # token 0 belongs to rank 0
    x = x.half().cuda()
    with torch.no_grad():
        y = lin(x)
    assert lin.state.idx.tolist() == [3, 200, 777]
    CB, SCB, _ = _state_of(lin)
    layers = _col_layers(CB, SCB, lin.bias.data, world, 6.0)
    Ms = M // world
    xs, CA, _, flags = layers[1].local_quantize(x[Ms:2 * Ms])
    assert not flags.any()  # rank 1 sees no outlier of its own
    assert (CA[:, [3, 200, 777]] != 0).any() or Ms == 1
    _check_col(x, y, CB, SCB, lin.bias.data, world, 6.0)


# ------------------------------------------------------------------------------------------ chain, world 1, graphs
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("M", [16, 256])
@pytest.mark.parametrize("threshold", [0.0, 6.0])
def test_sp_chain(world, M, threshold):
    """column(SP) -> GELU -> row(SP) gives the token rows of Linear8bitLt -> GELU -> Linear8bitLt."""
    import bitsandbytes_b200 as bnb
    from bitsandbytes_b200.parallel import _state_of

    H, I = 1024, 2048
    g = torch.Generator().manual_seed(M + world)
    up = bnb.nn.Linear8bitLt(H, I, bias=True, has_fp16_weights=False, threshold=threshold)
    down = bnb.nn.Linear8bitLt(I, H, bias=True, has_fp16_weights=False, threshold=threshold)
    with torch.no_grad():
        for lin, k in ((up, H), (down, I)):
            lin.weight.data = (torch.randn(lin.weight.shape, generator=g) / k**0.5).to(torch.float16)
            lin.bias.data = torch.randn(lin.bias.shape, generator=g).to(torch.float16)
    up, down = up.cuda().eval(), down.cuda().eval()
    x = torch.randn(M, H, generator=g)
    x[::5, [10, 500]] = 9.0
    x = x.to(torch.bfloat16).cuda()
    with torch.no_grad():
        want = down(torch.nn.functional.gelu(up(x)))
    (uCB, uSCB, _), (dCB, dSCB, _) = _state_of(up), _state_of(down)
    cols = _col_layers(uCB, uSCB, up.bias.data, world, threshold)
    rows = _row_layers(dCB, dSCB, down.bias.data, world, threshold, input_is_parallel=True)
    Ms = M // world
    for route in ("stage", "fused"):
        h = [torch.nn.functional.gelu(o) for o in _col_sp(cols, x, route)]
        outs = _row_sp(rows, h, route)
        torch.cuda.synchronize()
        for r, o in enumerate(outs):
            assert torch.equal(o, want[r * Ms:(r + 1) * Ms]), f"{route}, rank {r}"


@pytest.mark.parametrize("kind", ["col", "row"])
@pytest.mark.parametrize("threshold", [0.0, 6.0])
def test_world_one_sp_is_linear8bitlt(kind, threshold):
    from bitsandbytes_b200.parallel import ColumnParallelLinear8bitLt, RowParallelLinear8bitLt

    x, lin, y, _, _, _ = _reference(48, torch.float16, True, threshold, _outlier_cols(70, "spread") if threshold else (),
                                    seed=9)
    if kind == "col":
        layer = ColumnParallelLinear8bitLt.from_linear8bitlt(lin, gather_output=False, sequence_parallel=True)
    else:
        layer = RowParallelLinear8bitLt.from_linear8bitlt(lin, input_is_parallel=False, sequence_parallel=True)
    got = layer(x.view(6, 8, K_))
    assert got.shape == (6, 8, N_) and torch.equal(got.view(48, N_), y)


def test_threshold_zero_fused_sp_routes_replay_in_a_cuda_graph():
    """The fused SP column (code copies) and row (scatter GEMM) routes of four ranks, captured once and replayed on new
    inputs: the eager bits."""
    x, _, _, CB, SCB, bias = _reference(64, torch.bfloat16, True, 0.0, seed=12)
    cols = _col_layers(CB, SCB, bias, 4, 0.0)
    rows = _row_layers(CB, SCB, bias, 4, 0.0)
    static_x = x.clone()

    def step():
        return _col_sp(cols, static_x, "fused") + _row_sp(rows, [static_x] * 4, "fused")

    step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for seed in range(3):
        xn = (torch.randn(64, K_, generator=torch.Generator().manual_seed(200 + seed)) * 0.5).to(torch.bfloat16).cuda()
        static_x.copy_(xn)
        graph.replay()
        eager = step()
        torch.cuda.synchronize()
        for a, b in zip(outs, eager):
            assert torch.equal(a, b)


@pytest.mark.parametrize("kind", ["col", "row"])
def test_capture_with_threshold_raises(kind):
    x, _, _, CB, SCB, bias = _reference(16, torch.float16, False, 6.0, seed=3)
    layer = (_col_layers if kind == "col" else _row_layers)(CB, SCB, bias, 2, 6.0)[0]
    run = (lambda: layer.local_quantize(x[:8])) if kind == "col" else (lambda: layer.local_stats(layer.local_input(x)))
    run()  # eager is fine
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="capture"):
        with torch.cuda.graph(graph):
            run()


# ------------------------------------------------------------------------------------------ processes
_SCRIPT = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import bitsandbytes_b200 as bnb
from bitsandbytes_b200.parallel import (ColumnParallelLinear8bitLt, PeerInt8Input, PeerPartials,
                                        RowParallelLinear8bitLt, fused_forward_col8_sp, fused_forward_row8_sp)
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
H, I = 1024, 2048
for M, thr, J in ((8, 0.0, 0), (48, 6.0, 5), (256, 6.0, 80)):
    torch.manual_seed(0)
    up = bnb.nn.Linear8bitLt(H, I, bias=True, has_fp16_weights=False, threshold=thr)
    dn = bnb.nn.Linear8bitLt(I, H, bias=True, has_fp16_weights=False, threshold=thr)
    up.weight.data = (torch.randn(I, H) / H**0.5).half()
    dn.weight.data = (torch.randn(H, I) / I**0.5).half()
    up, dn = up.to(dev).eval(), dn.to(dev).eval()
    x = (torch.randn(M, H, device=dev) * 0.5).to(torch.bfloat16)
    x[::3, torch.arange(J, device=dev) * (H // max(J, 1))] = 7.0
    with torch.no_grad():
        hidden = up(x)
        want = dn(torch.nn.functional.gelu(hidden))
    Ms, Is = M // world, I // world
    xs = x[rank * Ms:(rank + 1) * Ms].contiguous()
    col = ColumnParallelLinear8bitLt.from_linear8bitlt(up, gather_output=False, sequence_parallel=True)
    row = RowParallelLinear8bitLt.from_linear8bitlt(dn, sequence_parallel=True)
    h = col(xs)
    assert torch.equal(h, hidden[:, rank * Is:(rank + 1) * Is]), f"M={M}: SP column (NCCL) differs"
    g = torch.nn.functional.gelu(h)
    y = row(g)
    assert torch.equal(y, want[rank * Ms:(rank + 1) * Ms]), f"M={M}: SP row (NCCL) differs"
    codes, parts = PeerInt8Input(M, H, dev), PeerPartials(Ms, H, dev, dtype=torch.int32)
    for _ in range(3):
        hf = fused_forward_col8_sp(col, xs, codes)
        yf = fused_forward_row8_sp(row, torch.nn.functional.gelu(hf), parts)
        torch.cuda.synchronize()
        assert torch.equal(hf, h), f"M={M}: fused SP column differs from NCCL SP"
        assert torch.equal(yf, y), f"M={M}: fused SP row differs from NCCL SP"
dist.barrier()
dist.destroy_process_group()
print("INT8_SP_OK", rank)
"""


@pytest.mark.parametrize("nproc", [1, 2])
def test_processes_fused_equals_nccl(tmp_path, nproc):
    """One process per GPU: the SP MLP through symmetric memory and through NCCL give Linear8bitLt's bits (the rank's
    feature columns, then its token rows) on every rank.  One process exercises the symmetric-memory routes; two need
    two GPUs."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "int8_sp.py"
    script.write_text(_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29601 + nproc), str(script)],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and r.stdout.count("INT8_SP_OK") == nproc, r.stdout[-2000:] + r.stderr[-3000:]
