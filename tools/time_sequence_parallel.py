"""Time the kernels of a sequence-parallel Linear4bit rank on one GPU against the non-SP ones, for the Llama-70B
down_proj (N = 8192, K = 28672) split over 8 GPUs (K = 3584 per rank), NF4, bf16:

  * the partial GEMM of the rank's K shard to one destination (the non-SP layer) and scattered over `--world` local
    buffers (the SP layer's fused route stores into the peers' buffers instead);
  * the rank-order reduction of `world` partials of [M, N] (non-SP) and of [M/world, N] (SP);
  * the SP column layer's `world` copies of a [M/world, K] token shard into local [M, K] buffers, at K = 8192.

CUDA events around `--iters` back-to-back launches, after `--warmup` of the same.  One JSON line per (M, kernel), then
the card's name and power limit (read, never set).

    python tools/time_sequence_parallel.py [--world 8] [--iters 200] [--warmup 20] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bitsandbytes_b200.functional as F  # noqa: E402
from bitsandbytes_b200.backends.cuda import gemm_4bit_partial, gemm_4bit_partial_scatter, reduce_partials  # noqa: E402
from bitsandbytes_b200.parallel import slice_quantized_weight_k  # noqa: E402


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e3 / iters  # us


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--tokens", type=int, nargs="+", default=[16, 256, 1024, 4096])
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda")
    N, K, w = 8192, 28672, a.world
    torch.manual_seed(0)
    W = (torch.randn(N, K, device=dev) / K**0.5).to(torch.bfloat16)
    qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="nf4")
    del W
    s = slice_quantized_weight_k(qW, qs, w, 0)
    Kc = 8192  # the column layer's input width (the hidden size)
    rows = []
    for M in a.tokens:
        Ms = M // w
        x = torch.randn(M, s.K, device=dev, dtype=torch.bfloat16)
        one = torch.empty((M, N), device=dev)
        scat = [torch.empty((Ms, N), device=dev) for _ in range(w)]
        stage = torch.randn((w, M, N), device=dev)
        stage_sp = torch.randn((w, Ms, N), device=dev)
        y = torch.empty((M, N), device=dev, dtype=torch.bfloat16)
        y_sp = torch.empty((Ms, N), device=dev, dtype=torch.bfloat16)
        bias = torch.randn(N, device=dev, dtype=torch.bfloat16)
        shard = torch.randn((Ms, Kc), device=dev, dtype=torch.bfloat16)
        gathered = [torch.empty((M, Kc), device=dev, dtype=torch.bfloat16) for _ in range(w)]

        def partial():
            gemm_4bit_partial(x, s.packed, (N, s.K), s.absmax, 64, "nf4", None, None, None, [one], N)

        def scatter():
            gemm_4bit_partial_scatter(x, s.packed, (N, s.K), s.absmax, 64, "nf4", None, None, None, scat, N)

        def reduce():
            reduce_partials(stage, torch.bfloat16, bias, out=y)

        def reduce_sp():
            reduce_partials(stage_sp, torch.bfloat16, bias, out=y_sp)

        def copies():
            for g in gathered:
                g[0:Ms].copy_(shard)

        weight_bytes = N * s.K // 2 + N * s.K // 64 * 4
        for name, fn, moved in (("partial_gemm_1_dest", partial, weight_bytes + 2 * M * s.K + 4 * M * N),
                                (f"partial_gemm_scatter_{w}_dests", scatter, weight_bytes + 2 * M * s.K + 4 * M * N),
                                (f"reduce_partials_{w}x[M,N]", reduce, 4 * w * M * N + 2 * M * N),
                                (f"reduce_partials_{w}x[M/{w},N]", reduce_sp, 4 * w * Ms * N + 2 * Ms * N),
                                (f"column_shard_copies_{w}x[M/{w},{Kc}]", copies, 2 * w * 2 * Ms * Kc)):
            if Ms == 0:
                continue
            us = timed(fn, a.iters, a.warmup)
            row = dict(kernel=name, M=M, N=N, K_shard=s.K, world=w, us=round(us, 2), bytes=moved,
                       GBps=round(moved / us / 1e3, 1))
            rows.append(row)
            print(json.dumps(row), flush=True)
        # the SP layer's output equals the non-SP rows bit for bit (same kernel): checked here on the timed shapes
        partial()
        scatter()
        torch.cuda.synchronize()
        assert torch.equal(torch.cat(scat), one), f"M={M}: scatter differs from the one-destination partial"
    info = card()
    print(json.dumps(dict(device=info)))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(device=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
