#!/usr/bin/env python
"""Per-rank kernel times of the tensor-parallel expert layers (CUDA events, one GPU).

    python tools/time_parallel_grouped.py --out DIR [--reps 20]

For one rank's shard (rank 0) at world sizes 1, 2, 4 and 8, on one GPU:

* ``column``: the column-parallel gate_up shard's grouped GEMM, ``[M, H] -> [M, 2 I / w]``
  (ColumnParallelGroupedLinear4bit.local_forward);
* ``row``: the row-parallel down shard's grouped fp32 partial ``[M, I / w] -> [M, H]`` into its slot of a
  ``[w, M, H]`` stage, plus the grouped reduction of the whole stage (RowParallelGroupedLinear4bit without the
  all-gather);
* ``unsharded``: GroupedLinear4bit's grouped GEMM on the whole gate_up and down weights, once per token count.

Each route's calls are captured in a CUDA graph and timed by replaying it, so the times are device times of the kernels
back to back, with no host dispatch inside the timed window.

The NCCL all-gathers between them need more than one GPU and are not measured here.  Shapes (NF4, blocksize 64, plain
statistics, bf16): Mixtral-8x22B (E 8, hidden 6144, intermediate 16384, top-2) and Qwen3-235B-A22B (E 128, hidden
4096, moe intermediate 1536, top-8), at 1, 16, 256 and 4096 tokens routed by a seeded top-k of uniform router scores.
Writes DIR/time_parallel_grouped.json and prints one JSON line per measurement, with the card's name, power limit and
maximum SM clock read in the same run.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

MODELS = (("mixtral_8x22b", 8, 6144, 16384, 2), ("qwen3_235b_a22b", 128, 4096, 1536, 8))
TOKENS = (1, 16, 256, 4096)
WORLDS = (1, 2, 4, 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()

    import torch

    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.backends.cuda import gemm_4bit_grouped_into, reduce_partials_grouped
    from bitsandbytes_b200.cextension import lib
    from bitsandbytes_b200.parallel import (ColumnParallelGroupedLinear4bit, RowParallelGroupedLinear4bit,
                                            slice_grouped_weight, slice_grouped_weight_k)

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")

    def timed(fn):
        """us per call of fn: `reps` calls captured in one CUDA graph (no host dispatch inside the timed window),
        warmed up eagerly and by one replay, then 5 replays between two events."""
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(args.reps):
                fn()
        graph.replay()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(5):
            graph.replay()
        b.record()
        torch.cuda.synchronize()
        lib.check("timed call")
        del graph
        return a.elapsed_time(b) * 1e3 / (5 * args.reps)

    def grouped_into(A, B, qs, offs, out):
        """GroupedLinear4bit's grouped GEMM on the whole weight, into a preallocated output."""
        gemm_4bit_grouped_into(A, B, tuple(qs.shape), qs.absmax, qs.blocksize, qs.quant_type, offs, None, None, None,
                               None, out, out.shape[1])

    def quantized(E, N, K):
        torch.manual_seed(0)
        W = (torch.randn(E, N, K, device=dev) / K**0.5).to(torch.bfloat16)
        return F.quantize_4bit(W, blocksize=64, quant_type="nf4")

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    rows = []

    def emit(**r):
        rows.append(r)
        print(json.dumps(r), flush=True)

    for name, E, H, I, topk in MODELS:
        gu, gu_qs = quantized(E, 2 * I, H)
        dn, dn_qs = quantized(E, H, I)
        for T in TOKENS:
            g = torch.Generator().manual_seed(T)
            choice = torch.rand(T, E, generator=g).topk(topk, dim=1).indices.reshape(-1)
            offs = torch.bincount(choice, minlength=E).cumsum(0).to(torch.int32).to(dev)
            M = T * topk
            x = torch.randn(M, H, device=dev, dtype=torch.bfloat16)
            a = torch.randn(M, I, device=dev, dtype=torch.bfloat16)
            base = dict(model=name, E=E, hidden=H, intermediate=I, tokens=T, rows=M)
            gu_out = torch.empty(M, 2 * I, device=dev, dtype=torch.bfloat16)
            dn_out = torch.empty(M, H, device=dev, dtype=torch.bfloat16)
            emit(**base, route="unsharded_gate_up", world=1,
                 us=round(timed(lambda: grouped_into(x, gu, gu_qs, offs, gu_out)), 2))
            emit(**base, route="unsharded_down", world=1,
                 us=round(timed(lambda: grouped_into(a, dn, dn_qs, offs, dn_out)), 2))
            del gu_out, dn_out
            for w in WORLDS:
                col = ColumnParallelGroupedLinear4bit(slice_grouped_weight(gu, gu_qs, w, 0), 2 * I)
                out = torch.empty(M, 2 * I // w, device=dev, dtype=torch.bfloat16)
                emit(**base, route="column", world=w,
                     us=round(timed(lambda: col.local_forward(x, out, out.shape[1], offs=offs)), 2))
                row = RowParallelGroupedLinear4bit(slice_grouped_weight_k(dn, dn_qs, w, 0), I)
                a_r = a[:, :I // w].contiguous()
                stage = torch.zeros(w, M, H, device=dev)
                y = torch.empty(M, H, device=dev, dtype=torch.bfloat16)
                emit(**base, route="row_partial", world=w,
                     us=round(timed(lambda: row.partial_forward(a_r, [stage[0]], offs=offs)), 2))
                emit(**base, route="row_reduce", world=w,
                     us=round(timed(lambda: reduce_partials_grouped(stage, offs, torch.bfloat16, out=y)), 2))
                del col, row, stage
                torch.cuda.empty_cache()
            emit(**base, route="nccl_exchange", world=None, us="not measured (needs more than one GPU)")
        del gu, dn
        torch.cuda.empty_cache()
    d = Path(args.out)
    d.mkdir(parents=True, exist_ok=True)
    (d / "time_parallel_grouped.json").write_text(json.dumps({"gpu": gpu, "reps": args.reps, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
