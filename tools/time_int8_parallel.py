"""Time the per-rank kernels of the tensor-parallel LLM.int8() layers on one GPU, at the Llama-70B world-8 shard shapes:
column (gate/up) 8192 -> 28672 / 8 and row (down_proj) 28672 / 8 -> 8192, against the unsharded Linear8bitLt GEMM of
the same rank's work (the column shard is an ordinary GEMM; for the row layer the reference is the fused GEMM over the
rank's K slice with fp16/bf16 output).  Kernels timed: the row statistics pass, the quantise-with-statistics pass, the
int32 partial GEMM, the int32 reduction of the world's partials (with J outlier columns), the column GEMM (with J
outlier columns), the fused GEMM over the row rank's K slice, and the whole unsharded layer's GEMM.  Sequence-parallel
rows from the same run: the int32 partial GEMM scattered over `world` destinations of M/world rows (against the
broadcast one), the reduction of `world` x [M/world, N] partials (against `world` x [M, N]), and the column layer's
quantisation of its M/world tokens plus `world` copies of their int8 codes (against quantising all M tokens; the copies
stand in for the stores into the peers' symmetric buffers and go to local memory here).  CUDA events around `--iters`
back-to-back launches after `--warmup`.
One JSON line per (shape, M, J, kernel), then the card's name and its power limit.  The NVLink exchange itself needs
two or more GPUs and is not measured here.

    python tools/time_int8_parallel.py [--world 8] [--iters 100] [--warmup 10] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bitsandbytes_b200.functional as F  # noqa: E402
from bitsandbytes_b200.backends.cuda import (int8_gemm_multi_out, int8_gemm_partial_scatter,  # noqa: E402
                                             int8_outlier_operands, int8_quant_with_stats, int8_reduce_partials,
                                             int8_row_stats, int8_vectorwise_quant_flags)


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


def power_limit() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--tokens", type=int, nargs="+", default=[16, 256, 1024, 4096])
    ap.add_argument("--outliers", type=int, nargs="+", default=[0, 5, 41])
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda")
    dt = torch.bfloat16
    torch.manual_seed(0)
    rows = []

    def emit(**row):
        rows.append(row)
        print(json.dumps(row), flush=True)

    # (name, N of the rank's GEMM, K of the rank's GEMM, full K)
    for shape, N, K, Nf, Kf in (("column_8192_to_28672", 28672 // a.world, 8192, 28672, 8192),
                                ("row_28672_to_8192", 8192, 28672 // a.world, 8192, 28672)):
        # the unsharded layer's GEMM on one GPU, threshold 0
        CBf = torch.randint(-127, 128, (Nf, Kf), device=dev, dtype=torch.int8)
        SCBf = torch.rand(Nf, device=dev) + 0.5
        for M in a.tokens:
            CAf, SCAf, _ = F.int8_vectorwise_quant(torch.randn(M, Kf, device=dev, dtype=torch.float16))
            yf = torch.empty((M, Nf), device=dev, dtype=dt)
            us = timed(lambda: int8_gemm_multi_out(CAf, CBf, SCAf, SCBf, [yf], Nf, dt), a.iters, a.warmup)
            emit(kernel="unsharded_linear8bitlt_gemm", shape=shape, M=M, N=Nf, K=Kf, us=round(us, 2),
                 TFLOPS=round(2.0 * M * Nf * Kf / us / 1e6, 1))
        del CBf
        CB = torch.randint(-127, 128, (N, K), device=dev, dtype=torch.int8)
        SCB = torch.rand(N, device=dev) + 0.5
        bias = torch.randn(N, device=dev, dtype=dt)
        for M in a.tokens:
            x = torch.randn(M, K, device=dev, dtype=dt)
            x16 = x.half()
            CA, SCA, _ = F.int8_vectorwise_quant(x16)
            y = torch.empty((M, N), device=dev, dtype=dt)
            parts = torch.randint(-2**20, 2**20, (a.world, M, N), device=dev, dtype=torch.int32)
            Ms = M // a.world
            sp = M % a.world == 0
            parts_sp = parts[:, :Ms].contiguous()
            for J in a.outliers:
                cols = torch.arange(J, device=dev) * (K // max(J, 1))
                subA = subBT = None
                if J:
                    subA, subBT = int8_outlier_operands(x, CB, SCB, cols)
                gemm_flops = 2.0 * M * N * K
                common = dict(shape=shape, M=M, N=N, K=K, world=a.world, J=J)

                def fused():
                    int8_gemm_multi_out(CA, CB, SCA, SCB, [y], N, dt, bias, subA, subBT)

                us = timed(fused, a.iters, a.warmup)
                emit(kernel="row_shard_fused_gemm" if shape.startswith("row") else "column_gemm", us=round(us, 2),
                     TFLOPS=round(gemm_flops / us / 1e6, 1), **common)
                if shape.startswith("row"):
                    def reduce():
                        int8_reduce_partials(parts, SCA, SCB, dt, bias, subA, subBT, out=y)

                    us = timed(reduce, a.iters, a.warmup)
                    moved = 4 * a.world * M * N + 2 * M * N
                    emit(kernel="int8_reduce_partials", us=round(us, 2), GBps=round(moved / us / 1e3, 1), **common)
                    if sp:
                        def reduce_sp():
                            int8_reduce_partials(parts_sp, SCA[:Ms], SCB, dt, bias, None if subA is None else subA[:Ms],
                                                 subBT, out=y[:Ms])

                        us = timed(reduce_sp, a.iters, a.warmup)
                        moved = 4 * a.world * Ms * N + 2 * Ms * N
                        emit(kernel="int8_reduce_partials_sp", us=round(us, 2), GBps=round(moved / us / 1e3, 1),
                             **common)
            if shape.startswith("row"):
                part = torch.empty((M, N), device=dev, dtype=torch.int32)

                def partial():
                    int8_gemm_multi_out(CA, CB, None, None, [part], N, None)

                def stats():
                    int8_row_stats(x16, 6.0)

                sca = torch.rand(M, device=dev) + 1

                def codes():
                    int8_quant_with_stats(x16, sca, 6.0)

                common = dict(shape=shape, M=M, N=N, K=K, world=a.world)
                us = timed(partial, a.iters, a.warmup)
                emit(kernel="int32_partial_gemm", us=round(us, 2), TFLOPS=round(2.0 * M * N * K / us / 1e6, 1),
                     **common)
                emit(kernel="row_stats", us=round(timed(stats, a.iters, a.warmup), 2), **common)
                emit(kernel="quant_with_stats", us=round(timed(codes, a.iters, a.warmup), 2), **common)
                if sp:
                    scat = [torch.empty((Ms, N), device=dev, dtype=torch.int32) for _ in range(a.world)]

                    def partial_scatter():
                        int8_gemm_partial_scatter(CA, CB, scat, N)

                    us = timed(partial_scatter, a.iters, a.warmup)
                    emit(kernel="int32_partial_gemm_scatter", us=round(us, 2),
                         TFLOPS=round(2.0 * M * N * K / us / 1e6, 1), **common)
            elif sp:
                # the column layer's input side: K is the full input width here
                gathered = torch.empty((M, K), device=dev, dtype=torch.int8)

                def quant_all():
                    int8_vectorwise_quant_flags(x16, 6.0)

                def quant_sp():
                    CAs, _, _ = int8_vectorwise_quant_flags(x16[:Ms], 6.0)
                    for r in range(a.world):
                        gathered[r * Ms:(r + 1) * Ms].copy_(CAs)

                common = dict(shape=shape, M=M, K=K, world=a.world)
                emit(kernel="quantize_all_tokens", us=round(timed(quant_all, a.iters, a.warmup), 2), **common)
                emit(kernel="quantize_sp_tokens_and_copy_codes", us=round(timed(quant_sp, a.iters, a.warmup), 2),
                     **common)
    info = dict(device=torch.cuda.get_device_name(), power_limit=power_limit(), nvlink_exchange="not measured")
    print(json.dumps(info))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
