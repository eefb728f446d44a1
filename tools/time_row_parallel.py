"""Time the two kernels of a row-parallel Linear4bit rank on one GPU: the partial 4-bit GEMM of the rank's K shard
(fp32 accumulators, no bias) and the rank-order reduction of the world's partials, for the Llama-70B down_proj
(N = 8192, K = 28672) split over 8 GPUs (K = 3584 per rank), NF4, bf16.  Beside them: the plain GEMM of the same shard
(bf16 output), to show what the fp32 output costs, and the bytes each kernel moves.  CUDA events around `--iters`
back-to-back launches, after `--warmup` of the same.  One JSON line per (M, kernel), then the card's name.

    python tools/time_row_parallel.py [--world 8] [--iters 200] [--warmup 20] [--out result.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bitsandbytes_b200.functional as F  # noqa: E402
from bitsandbytes_b200.backends.cuda import gemm_4bit_into, gemm_4bit_partial, reduce_partials  # noqa: E402
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--tokens", type=int, nargs="+", default=[1, 16, 256, 1024, 4096])
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda")
    N, K = 8192, 28672
    torch.manual_seed(0)
    W = (torch.randn(N, K, device=dev) / K**0.5).to(torch.bfloat16)
    qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="nf4")
    del W
    s = slice_quantized_weight_k(qW, qs, a.world, 0)
    rows = []
    for M in a.tokens:
        x = torch.randn(M, s.K, device=dev, dtype=torch.bfloat16)
        stage = torch.empty((a.world, M, N), device=dev, dtype=torch.float32)
        stage.normal_()
        y = torch.empty((M, N), device=dev, dtype=torch.bfloat16)
        bias = torch.randn(N, device=dev, dtype=torch.bfloat16)

        def partial():
            gemm_4bit_partial(x, s.packed, (N, s.K), s.absmax, 64, "nf4", None, None, None, [stage[0]], N)

        def plain():
            gemm_4bit_into(x, s.packed, (N, s.K), s.absmax, 64, "nf4", None, None, None, None, y, N)

        def reduce():
            reduce_partials(stage, torch.bfloat16, bias, out=y)

        weight_bytes = N * s.K // 2 + N * s.K // 64 * 4
        for name, fn, moved in (("partial_gemm", partial, weight_bytes + 2 * M * s.K + 4 * M * N),
                                ("plain_gemm_bf16_out", plain, weight_bytes + 2 * M * s.K + 2 * M * N),
                                ("reduce_partials", reduce, 4 * a.world * M * N + 2 * M * N)):
            us = timed(fn, a.iters, a.warmup)
            row = dict(kernel=name, M=M, N=N, K_shard=s.K, world=a.world, us=round(us, 2),
                       bytes=moved, GBps=round(moved / us / 1e3, 1))
            if name != "reduce_partials":
                row["TFLOPS"] = round(2.0 * M * N * s.K / us / 1e6, 1)
            rows.append(row)
            print(json.dumps(row), flush=True)
    name = torch.cuda.get_device_name()
    print(json.dumps(dict(device=name)))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(device=name, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
