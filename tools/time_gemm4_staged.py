#!/usr/bin/env python
"""Phase timings of the staged 4-bit GEMM route against the fused kernel and cuBLAS (CUDA events, one H100).

    python tools/time_gemm4_staged.py --out DIR [--reps 50]

For each benchmark weight shape (4096x4096, 11008x4096, 4096x11008; NF4, blocksize 64, bf16) and M in
{512, 1024, 2048, 4096}: the dequantise pass alone (every panel of the weight), the staged GEMM alone on a decoded
weight, the whole staged route, the fused kernel (its production token tile and K split) and cuBLAS bf16 on the
decoded weight.  Then the whole route at M = 4096 for several panel sizes.  Writes DIR/time_gemm4_staged.json and
prints one line per measurement.  The crossover M where the route beats the fused kernel sets kStagedMinM
(csrc/c_api.cu).
"""
import argparse
import ctypes as ct
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SHAPES = ((4096, 4096), (11008, 4096), (4096, 11008))
MS = (512, 1024, 2048, 4096)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()

    import torch

    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.cextension import lib

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")
    st = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731

    def timed(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        lib.check("timed call")
        return a.elapsed_time(b) * 1e3 / args.reps  # us per call

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = []
    for N, K in SHAPES:
        torch.manual_seed(0)
        W = (torch.randn(N, K, device=dev) / K**0.5).to(torch.bfloat16)
        qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="nf4")
        Wd = F.dequantize_4bit(qW, qs).contiguous()
        del W
        panel_max = max(128, (32 << 20) // (2 * K) // 128 * 128)
        for M in MS:
            x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
            out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            outs = (ct.c_void_p * 1)(out.data_ptr())

            def deq():
                for n0 in range(0, N, panel_max):
                    assert lib.cbnb_b200_dequantize_4bit_panel(qW.data_ptr(), qs.absmax.data_ptr(), None, None, None,
                                                               Wd.data_ptr(), 64, 2, 2, n0, min(panel_max, N - n0), K,
                                                               st()) == 0

            def gemm(mt):
                return lambda: lib.cbnb_b200_gemm_decoded(x.data_ptr(), Wd.data_ptr(), out.data_ptr(), None, M, N, K,
                                                          N, 2, mt, st())

            def route(panel=0):
                return lambda: lib.cbnb_b200_gemm_4bit_staged(x.data_ptr(), qW.data_ptr(), qs.absmax.data_ptr(), None,
                                                              None, None, ct.cast(outs, ct.c_void_p), 1, None, M, N,
                                                              K, N, 64, 2, 2, 0, panel, st())

            def fused():
                lib.cbnb_b200_gemm_4bit_pair(x.data_ptr(), qW.data_ptr(), qs.absmax.data_ptr(), None, None, None,
                                             out.data_ptr(), None, M, N, K, N, 64, 2, 2, 0, 0, None, st())

            r = {"N": N, "K": K, "M": M, "staged_route": lib.cbnb_b200_gemm_4bit_staged_route(M, N, K, 64, 2),
                 "dequant_us": timed(deq), "gemm_ss_mt256_us": timed(gemm(256)), "gemm_ss_mt128_us": timed(gemm(128)),
                 "route_us": timed(route()), "fused_us": timed(fused),
                 "cublas_bf16_us": timed(lambda: torch.matmul(x, Wd.t(), out=out))}
            if M == 4096:
                for pr in (512, 1024, 2048, panel_max):
                    if pr <= panel_max:
                        r[f"route_panel{pr}_us"] = timed(route(pr))
            r["tflops_route"] = 2.0 * M * N * K / r["route_us"] / 1e6
            rows.append(r)
            print(json.dumps(r), flush=True)
    d = Path(args.out)
    d.mkdir(parents=True, exist_ok=True)
    (d / "time_gemm4_staged.json").write_text(json.dumps({"gpu": gpu, "reps": args.reps, "rows": rows}, indent=1))
    print(gpu)


if __name__ == "__main__":
    main()
