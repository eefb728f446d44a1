"""GPU: the tensor-parallel expert layers (bitsandbytes_b200/parallel.py) and the two kernels under them.

* cbnb_b200_gemm_4bit_grouped_partial, every instance (dtype x quant type x token tile): the fp32 partial within the
  fp32 accumulation bound of a float64 product, exact zeros in the tail rows, and T(P + bias_e) equal to the grouped
  GEMM at the same tile bit for bit.
* cbnb_b200_reduce_partials_grouped: bit for bit a torch rank-order fp32 sum plus the row's expert bias, rounded once.
* The layers, simulated rank by rank at worlds 2, 4 and 8: the column layer's gathered output is GroupedLinear4bit's
  bit for bit; the row layer's is at world 1, and within the fp32 bound of the float64 product at larger worlds.
* A column -> SiLU.up -> row pair through the layers' own forwards and collectives, with the ranks as threads of one
  process and, on as many GPUs, as processes over NCCL: every rank's output equals the rank-by-rank simulation.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.backends.cuda as cb
import bitsandbytes_b200.functional as F
from bitsandbytes_b200.parallel import (ColumnParallelGroupedLinear4bit, RowParallelGroupedLinear4bit,
                                        slice_grouped_weight, slice_grouped_weight_k)
from tests import _native as nat

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
GUARD = 64


def clamp_ends(offs, M):
    ends, run = [], 0
    for o in offs:
        run = min(max(o, run), M)
        ends.append(run)
    return ends


def expert_of_rows(offs, M, device="cuda"):
    """(the expert of every row, -1 past the last end) for offs clamped as the kernels clamp them."""
    ends = clamp_ends(offs, M)
    e = torch.full((M,), -1, dtype=torch.long)
    start = 0
    for i, end in enumerate(ends):
        e[start:end] = i
        start = max(start, end)
    return e.to(device)


def quantized_experts(E, N, K, dtype, qt="nf4", bs=64, nested=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = (torch.randn(E, N, K, generator=g, device="cuda") / K**0.5).to(dtype)
    packed, qs = F.quantize_4bit(W, blocksize=bs, compress_statistics=nested, quant_type=qt)
    return packed, qs


def decoded(packed, qs, dtype):
    """The [E, N, K] weights as the kernels decode them."""
    return F.dequantize_4bit(packed, qs).to(dtype).reshape(qs.shape)


def fp32_bound(x, W, rows_expert, K):
    """K * 2^-23 * sum_k |x[m, k] W_e[n, k]|, per element: the bound of an fp32 sum of K exact products (two units of
    fp32 rounding per addition, which also covers an accumulator that truncates)."""
    xa = x.double().abs()
    bound = torch.zeros((x.shape[0], W.shape[1]), dtype=torch.float64, device=x.device)
    for e in range(W.shape[0]):
        rows = rows_expert == e
        if rows.any():
            bound[rows] = xa[rows] @ W[e].double().abs().T
    return bound * K * 2.0**-23


def assert_within_bound(y, y64, acc_bound, dtype):
    """y (rounded once to T) against the float64 value: the fp32 accumulation bound, one fp32 rounding of the bias
    addition, and half an ulp of T at the larger of the two magnitudes."""
    g = y.double()
    assert torch.isfinite(g).all()
    mag = torch.maximum(y64.abs(), g.abs())
    ulp = torch.exp2(torch.floor(torch.log2(mag.clamp(min=1e-30))) - (7 if dtype == "bf16" else 10))
    bound = acc_bound + 2.0**-23 * mag + 0.5 * ulp
    err = (g - y64).abs()
    assert (err <= bound).all(), f"max error {err.max().item()}, over the bound by {(err - bound).max().item()}"


def product64(x, W, rows_expert, bias=None):
    y = torch.zeros((x.shape[0], W.shape[1]), dtype=torch.float64, device=x.device)
    for e in range(W.shape[0]):
        rows = rows_expert == e
        if rows.any():
            y[rows] = x[rows].double() @ W[e].double().T
            if bias is not None:
                y[rows] += bias[e].double()
    return y


def grouped_partial(x, packed, absmax, offs_t, E, N, K, mt, ldc, bs=64, qt="nf4"):
    M = x.shape[0]
    buf = torch.full((M * ldc + GUARD,), float("nan"), device="cuda")
    out = buf[:M * ldc].view(M, ldc)[:, :N]
    rc = nat.lib.cbnb_b200_gemm_4bit_grouped_partial(x.data_ptr(), packed.data_ptr(), absmax.data_ptr(),
                                                     offs_t.data_ptr(), E, out.data_ptr(), M, N, K, ldc, bs,
                                                     nat.QT_ID[qt], nat.DTYPE_ID[{torch.bfloat16: "bf16",
                                                                                  torch.float16: "fp16"}[x.dtype]],
                                                     mt, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0, rc
    assert torch.isnan(buf[M * ldc:]).all(), "guard elements written"
    assert torch.isnan(buf[:M * ldc].view(M, ldc)[:, N:]).all(), "padding columns [N, ldc) written"
    return out


def grouped_mt(x, packed, absmax, offs_t, E, N, K, mt, bias, bs=64, qt="nf4"):
    M = x.shape[0]
    out = torch.full((M, N), float("nan"), dtype=x.dtype, device="cuda")
    rc = nat.lib.cbnb_b200_gemm_4bit_grouped_mt(x.data_ptr(), packed.data_ptr(), absmax.data_ptr(), None, None, None,
                                                offs_t.data_ptr(), E, out.data_ptr(), nat.ptr(bias), M, N, K, N, bs,
                                                nat.QT_ID[qt], nat.DTYPE_ID[{torch.bfloat16: "bf16",
                                                                             torch.float16: "fp16"}[x.dtype]],
                                                mt, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0, rc
    return out


# ---------------------------------------------------------------------------------------------------- the partial GEMM
ROUTINGS = {
    # an empty expert in the middle, counts below / not a multiple of the tile, tail rows
    "empty_and_tail": lambda mt: (np.cumsum([mt + 3, 0, 1, 2 * mt - 1]).tolist(), 3 * mt + 3 + 5),
    # offs below zero, decreasing and past M: clamped on the device, no tail
    "malformed": lambda mt: ([-3, mt + 7, 5, 10**6], 2 * mt + 9),
}


@pytest.mark.parametrize("routing", list(ROUTINGS))
@pytest.mark.parametrize("mt", [16, 32, 64, 128])
@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_every_partial_instance(dtype, qt, mt, routing):
    """N = 192, so that an expert's second n-tile reaches into the next expert's codes; ldc = N + 5 (strided)."""
    E, N, K = 4, 192, 512
    offs, M = ROUTINGS[routing](mt)
    T = DT[dtype]
    packed, qs = quantized_experts(E, N, K, T, qt, seed=mt)
    g = torch.Generator(device="cpu").manual_seed(mt + 1)
    x = torch.randn(M, K, generator=g).to(T).cuda()
    bias = torch.randn(E, N, generator=g).to(T).cuda()
    offs_t = torch.tensor(offs, dtype=torch.int32, device="cuda")
    P = grouped_partial(x, packed, qs.absmax, offs_t, E, N, K, mt, N + 5, qt=qt)
    rows_e = expert_of_rows(offs, M)
    tail = rows_e < 0
    assert (P[tail] == 0).all() and not torch.signbit(P[tail]).any(), "tail rows are not +0"
    W = decoded(packed, qs, T)
    err = (P.double() - product64(x, W, rows_e)).abs()
    assert (err <= fp32_bound(x, W, rows_e, K)).all(), f"max error {err.max().item()}"
    # T(P + bias_e), rounded once, is the grouped GEMM's epilogue
    want = grouped_mt(x, packed, qs.absmax, offs_t, E, N, K, mt, bias, qt=qt)
    be = torch.where(tail[:, None], torch.zeros_like(P), bias.float()[rows_e.clamp(min=0)])
    assert torch.equal((P + be).to(T), want)


def test_partial_default_tile_is_the_grouped_rule():
    """mt = 0 takes the grouped GEMM's tile rule, the one the unsharded layer takes."""
    E, N, K = 8, 128, 256
    offs = np.cumsum([40] * 8).tolist()
    packed, qs = quantized_experts(E, N, K, torch.bfloat16)
    x = torch.randn(320, K, device="cuda").to(torch.bfloat16)
    offs_t = torch.tensor(offs, dtype=torch.int32, device="cuda")
    P = grouped_partial(x, packed, qs.absmax, offs_t, E, N, K, 0, N)
    assert torch.equal(P.to(torch.bfloat16), grouped_mt(x, packed, qs.absmax, offs_t, E, N, K, 128, None))


def test_partial_refuses_without_writing():
    E, N, K = 2, 64, 96  # K % 64 != 0: not served
    x = torch.zeros(8, K, device="cuda", dtype=torch.bfloat16)
    B = torch.zeros(E * N * K // 2, dtype=torch.uint8, device="cuda")
    absmax = torch.ones(E * N * K // 32, device="cuda")
    offs = torch.tensor([4, 8], dtype=torch.int32, device="cuda")
    out = torch.full((8, N), float("nan"), device="cuda")
    rc = nat.lib.cbnb_b200_gemm_4bit_grouped_partial(x.data_ptr(), B.data_ptr(), absmax.data_ptr(), offs.data_ptr(),
                                                     E, out.data_ptr(), 8, N, K, N, 32, 2, 2, 0, nat.stream())
    torch.cuda.synchronize()
    assert rc == 100 and torch.isnan(out).all()
    rc = nat.lib.cbnb_b200_gemm_4bit_grouped_partial(x.data_ptr(), B.data_ptr(), absmax.data_ptr(), offs.data_ptr(),
                                                     E, out.data_ptr(), 8, N, 128, N - 1, 32, 2, 2, 0, nat.stream())
    assert rc == 1
    with pytest.raises(RuntimeError, match="gemm_4bit_grouped_partial"):
        nat.check()  # the message is set, and reading it clears it


# ---------------------------------------------------------------------------------------------------- the reduction
def reduce_ref(parts, offs, dtype, bias):
    world, M, N = parts.shape
    rows_e = expert_of_rows(offs, M)
    s = parts[0].clone()
    for r in range(1, world):
        s = s + parts[r]
    b = torch.zeros_like(s) if bias is None else bias.float()[rows_e.clamp(min=0)]
    s = s + b
    s[rows_e < 0] = 0
    return s.to(dtype)


@pytest.mark.parametrize("path", ["vector", "element"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 6, 7, 8])
def test_grouped_reduce_is_the_rank_order_sum(world, dtype, bias, path):
    T = DT[dtype]
    E, M = 5, 77
    N, ldc = (256, 264) if path == "vector" else (100, 101)
    g = torch.Generator(device="cpu").manual_seed(world * 10 + len(path))
    parts = (torch.randn(world, M, N, generator=g) * 4).cuda()
    offs = [10, 10, 33, 30, 70]  # an empty expert, a decreasing end, 7 tail rows
    b = torch.randn(E, N, generator=g).to(T).cuda() if bias else None
    buf = torch.full((M * ldc + GUARD,), float("nan"), dtype=T, device="cuda")
    out = buf[:M * ldc].view(M, ldc)[:, :N]
    got = cb.reduce_partials_grouped(parts, torch.tensor(offs, dtype=torch.int32, device="cuda"), T, b, out=out)
    torch.cuda.synchronize()
    assert torch.equal(got, reduce_ref(parts, offs, T, b))
    assert torch.isnan(buf[M * ldc:]).all()
    assert torch.isnan(buf[:M * ldc].view(M, ldc)[:, N:]).all(), "padding columns written"
    if not bias:  # no bias, and no tail: the plain reduction's bits
        full = torch.tensor([10, 20, 40, 60, M], dtype=torch.int32, device="cuda")
        assert torch.equal(cb.reduce_partials_grouped(parts, full, T), cb.reduce_partials(parts, T))


# ---------------------------------------------------------------------------------------------------- the layers
def column_sim(packed, qs, world, x, offs_t, bias):
    """The gathered output of a column layer, rank by rank: each simulated rank's shard runs ``local_forward``, which
    consults no process group, so the simulation gives the same result inside an initialised one."""
    cols = []
    for r in range(world):
        layer = ColumnParallelGroupedLinear4bit(slice_grouped_weight(packed, qs, world, r), qs.shape[1], bias,
                                                gather_output=False)
        cols.append(layer.local_forward(x, offs=offs_t))
    return torch.cat(cols, dim=1)


def row_sim(packed, qs, world, x, offs_t, bias):
    """The output of a row layer, rank by rank: every rank's partial into its slot, then the grouped reduction."""
    E, N, K = qs.shape
    parts = torch.empty((world, x.shape[0], N), device="cuda")
    for r in range(world):
        layer = RowParallelGroupedLinear4bit(slice_grouped_weight_k(packed, qs, world, r), K, bias,
                                             input_is_parallel=False)
        layer.partial_forward(layer.local_input(x), [parts[r]], offs=offs_t)
    return cb.reduce_partials_grouped(parts, offs_t, x.dtype, bias)


def grouped_ref(x, packed, qs, offs_t, bias):
    return bnb.grouped_matmul_4bit(x, packed, qs, offs_t, bias=bias)


def pair_problem():
    """A gate_up [8, 2048, 512] and down [8, 512, 1024] expert pair with biases, 160 routed rows and their offs: the same
    tensors in every process (seeded)."""
    E, H, I = 8, 512, 1024
    T = torch.bfloat16
    gu, gu_qs = quantized_experts(E, 2 * I, H, T, seed=1)
    dn, dn_qs = quantized_experts(E, H, I, T, seed=2)
    g = torch.Generator(device="cpu").manual_seed(7)
    gu_b = torch.randn(E, 2 * I, generator=g).to(T).cuda()
    dn_b = torch.randn(E, H, generator=g).to(T).cuda()
    x = torch.randn(160, H, generator=g).to(T).cuda()
    offs = torch.tensor([10, 10, 40, 80, 81, 120, 150, 155], dtype=torch.int32, device="cuda")
    return dict(gu=gu, gu_qs=gu_qs, gu_b=gu_b, dn=dn, dn_qs=dn_qs, dn_b=dn_b, x=x, offs=offs)


def gated(h, world):
    """SiLU(gate) * up of each rank's [gate | up] halves of the column output h [M, world * w] (a gate_up tensor whose
    rows are ordered rank by rank), rank after rank."""
    w = h.shape[1] // world
    return torch.cat([torch.nn.functional.silu(h[:, r * w:r * w + w // 2]) * h[:, r * w + w // 2:(r + 1) * w]
                      for r in range(world)], dim=1)


def pair_on_rank(p):
    """This rank's column -> SiLU.up -> row forward, through the layers and their collectives (the process group's world
    and rank, as _group_world_rank reports them)."""
    col = ColumnParallelGroupedLinear4bit.from_quantized(p["gu"], p["gu_qs"], p["gu_b"], gather_output=False)
    row = RowParallelGroupedLinear4bit.from_quantized(p["dn"], p["dn_qs"], p["dn_b"])
    return row(gated(col(p["x"], p["offs"]), 1), p["offs"])


def pair_simulated(p, world):
    """The same pair, every rank simulated in turn with no collective."""
    hs = column_sim(p["gu"], p["gu_qs"], world, p["x"], p["offs"], p["gu_b"])
    return row_sim(p["dn"], p["dn_qs"], world, gated(hs, world), p["offs"], p["dn_b"])


@pytest.mark.parametrize("world", [2, 4, 8])
def test_ranks_as_threads_equal_the_simulation(monkeypatch, world):
    """The layers' own forwards, collectives included, with each rank a thread of this process: the all-gather is a
    barrier across the threads that hands every rank all ranks' slots.  Every rank's output equals the rank-by-rank
    simulation bit for bit (the NCCL route's logic, on one GPU)."""
    import threading

    import bitsandbytes_b200.parallel as par

    p = pair_problem()
    local = threading.local()
    barrier = threading.Barrier(world, timeout=120)
    slots = {}

    def all_gather_into_tensor(out, inp, group=None):
        torch.cuda.synchronize()  # this rank's slot is complete
        slots[local.rank] = inp
        barrier.wait()
        out.view(world, -1).copy_(torch.stack([slots[r].reshape(-1) for r in range(world)]))
        torch.cuda.synchronize()
        barrier.wait()  # every rank has copied before a slot is published again

    monkeypatch.setattr(par, "_group_world_rank", lambda group: (world, local.rank))
    monkeypatch.setattr(par.dist, "all_gather_into_tensor", all_gather_into_tensor)
    want = pair_simulated(p, world)  # inside the patched world, as in a process of an initialised group
    got, errors = {}, []

    def rank_main(r):
        local.rank = r
        try:
            got[r] = pair_on_rank(p)
            torch.cuda.synchronize()
        except BaseException as e:  # reported below; the barrier's timeout releases the other ranks
            errors.append((r, e))
            barrier.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for r in range(world):
        assert torch.equal(got[r], want), f"rank {r}"


COLUMN_CASES = {
    "plain": dict(E=4, N=512, K=512, nested=False),
    "nested_kept": dict(E=4, N=512, K=512, nested=True),          # 512/w rows * 8 blocks: whole 256-block groups
    "nested_converted": dict(E=3, N=384, K=320, nested=True),     # per-expert slices off the 256-block grid
}


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("case", list(COLUMN_CASES))
def test_column_layer_equals_grouped_linear(case, world):
    c = COLUMN_CASES[case]
    E, N, K = c["E"], c["N"], c["K"]
    packed, qs = quantized_experts(E, N, K, torch.bfloat16, nested=c["nested"], seed=world)
    kept = [slice_grouped_weight(packed, qs, world, r).absmax_8bit is not None for r in range(world)]
    if case == "nested_kept":
        assert all(kept)
    if case == "nested_converted":
        assert not any(kept)
    x = torch.randn(150, K, device="cuda").to(torch.bfloat16)
    offs_t = torch.tensor(np.cumsum([30, 0, 70, 40][:E]).tolist()[:E], dtype=torch.int32, device="cuda")
    bias = torch.randn(E, N, device="cuda").to(torch.bfloat16)
    assert torch.equal(column_sim(packed, qs, world, x, offs_t, bias), grouped_ref(x, packed, qs, offs_t, bias))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_row_layer(world, dtype):
    """World 1: GroupedLinear4bit bit for bit.  Larger worlds: within the fp32 bound of the float64 product (each
    rank's partial and the rank-order sum together are an fp32 sum of K exact products), plus the final rounding."""
    T = DT[dtype]
    E, N, K = 6, 256, 2048
    packed, qs = quantized_experts(E, N, K, T, nested=True, seed=world)
    offs = [20, 20, 91, 60, 140, 190]
    M = 201
    x = torch.randn(M, K, device="cuda").to(T)
    offs_t = torch.tensor(offs, dtype=torch.int32, device="cuda")
    bias = torch.randn(E, N, device="cuda").to(T)
    y = row_sim(packed, qs, world, x, offs_t, bias)
    if world == 1:
        assert torch.equal(y, grouped_ref(x, packed, qs, offs_t, bias))
    rows_e = expert_of_rows(offs, M)
    W = decoded(packed, qs, T)
    y64 = product64(x, W, rows_e, bias)
    y64[rows_e < 0] = 0
    assert_within_bound(y, y64, fp32_bound(x, W, rows_e, K), dtype)


def test_cuda_graph_replays_new_routings():
    """A world-1 column -> SiLU-up -> row pair captured once; replays with new routings written into offs in place give
    the eager outputs bit for bit."""
    E, H, I = 8, 512, 1024
    T = torch.bfloat16
    gu_packed, gu_qs = quantized_experts(E, 2 * I, H, T, seed=1)
    dn_packed, dn_qs = quantized_experts(E, H, I, T, seed=2)
    col = ColumnParallelGroupedLinear4bit.from_quantized(gu_packed, gu_qs, torch.randn(E, 2 * I, device="cuda").to(T))
    row = RowParallelGroupedLinear4bit.from_quantized(dn_packed, dn_qs, torch.randn(E, H, device="cuda").to(T))
    M = 96
    x = torch.randn(M, H, device="cuda").to(T)
    offs = torch.zeros(E, dtype=torch.int32, device="cuda")

    def step():
        h = col(x, offs)
        return row(torch.nn.functional.silu(h[:, :I]) * h[:, I:], offs)

    routings = [[12] * 8, [0, 0, 50, 50, 90, 90, 90, 96], [96] * 8, [5, 3, 80, 200, -1, 7, 9, 11]]
    offs.copy_(torch.tensor(routings[0], dtype=torch.int32))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()  # warm-up: allocates the layers' stages outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = step()
    for r in routings:
        offs.copy_(torch.tensor(r, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, step())


# ---------------------------------------------------------------------------------------------------- real shapes
def top_k_offs(tokens, E, k, seed):
    """End rows of the expert-sorted rows of `tokens` tokens routed top-k at random."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    choice = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(tokens)]).reshape(-1)
    return torch.cumsum(torch.bincount(choice, minlength=E), 0).to(torch.int32).cuda()


def test_qwen3_235b_down_layer_at_world_4():
    """Qwen3-235B-A22B's down projection (128 experts, moe intermediate 1536 -> hidden 4096) at w = 4, 64 tokens
    top-8: every rank simulated; within the fp32 bound of the float64 product."""
    E, N, K, w = 128, 4096, 1536, 4
    packed, qs = quantized_experts(E, N, K, torch.bfloat16, nested=True, seed=3)
    offs_t = top_k_offs(64, E, 8, 3)
    M = 64 * 8
    x = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    y = row_sim(packed, qs, w, x, offs_t, None)
    rows_e = expert_of_rows(offs_t.tolist(), M)
    W = decoded(packed, qs, torch.bfloat16)
    assert_within_bound(y, product64(x, W, rows_e), fp32_bound(x, W, rows_e, K), "bf16")


def test_mixtral_8x22b_gate_up_layer_at_world_8():
    """Mixtral-8x22B's gate_up projection (8 experts, hidden 6144 -> 2 x 16384) at w = 8, 256 tokens top-2: the
    gathered output of the 8 simulated ranks is GroupedLinear4bit's bit for bit."""
    E, N, K, w = 8, 2 * 16384, 6144, 8
    packed, qs = quantized_experts(E, N, K, torch.bfloat16, nested=True, seed=4)
    offs_t = top_k_offs(256, E, 2, 4)
    x = torch.randn(512, K, device="cuda").to(torch.bfloat16)
    assert torch.equal(column_sim(packed, qs, w, x, offs_t, None), grouped_ref(x, packed, qs, offs_t, None))


# ---------------------------------------------------------------------------------------------------- processes
_SCRIPT = r"""
import os, sys
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import torch
import torch.distributed as dist
from tests.test_gpu_parallel_grouped import pair_on_rank, pair_problem, pair_simulated

dist.init_process_group("nccl")
rank, world = dist.get_rank(), dist.get_world_size()
torch.cuda.set_device(rank)
p = pair_problem()
y = pair_on_rank(p)
want = pair_simulated(p, world)
assert torch.equal(y, want), (y.float() - want.float()).abs().max()
dist.barrier()
dist.destroy_process_group()
print("GROUPED_TP_OK", rank)
"""


@pytest.mark.parametrize("nproc", [1, 2, 4])
def test_processes_column_row_pair_equals_simulation(tmp_path, nproc):
    """One process per GPU over NCCL: a column -> SiLU.up -> row pair equals the rank-by-rank simulation bit for bit."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "grouped_tp.py"
    script.write_text(_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29771 + nproc), str(script)],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and r.stdout.count("GROUPED_TP_OK") == nproc, r.stdout[-3000:] + r.stderr[-4000:]
