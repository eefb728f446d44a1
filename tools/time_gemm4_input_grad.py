#!/usr/bin/env python
"""Timings of the input-gradient 4-bit GEMM (out = G . dequant(W)) against dequantise + torch.matmul (CUDA events).

    python tools/time_gemm4_input_grad.py --out DIR [--reps 30]

Weights (N x K, NF4, blocksize 64, bf16): the shards of the tensor-parallel benchmark (3584 x 8192 column, 8192 x 3584
row) and the Llama-3-8B projections (4096 x 4096, 14336 x 4096, 4096 x 14336), at M in {256, 2048, 4096}.  For each:
the kernel's T output (bf16) and its fp32 output (the partial of a column-parallel layer), against dequantize_4bit +
torch.matmul giving bf16, dequantize_4bit + cuBLAS on the bf16 operands with an fp32 output
(torch.mm(..., out_dtype=torch.float32), the other route to an fp32 partial), and dequantize_4bit + an fp32 matmul on
fp32 copies.
Writes DIR/time_gemm4_input_grad.json, with the card's name and power limit read in the same run, and prints one line
per shape.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SHAPES = ((3584, 8192), (8192, 3584), (4096, 4096), (14336, 4096), (4096, 14336))
MS = (256, 2048, 4096)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()

    import torch

    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.backends.cuda import gemm_4bit_input_grad
    from bitsandbytes_b200.cextension import lib

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")

    def timed(fn):
        for _ in range(3):
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
        del W
        for M in MS:
            G = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
            t_out = torch.empty(M, K, device=dev, dtype=torch.bfloat16)
            p_out = torch.empty(M, K, device=dev)

            def kernel(out):
                assert gemm_4bit_input_grad(G, qW, (N, K), qs.absmax, 64, "nf4", None, None, None, out)

            r = {"N": N, "K": K, "M": M,
                 "kernel_T_us": timed(lambda: kernel(t_out)),
                 "kernel_fp32_us": timed(lambda: kernel(p_out)),
                 "dequant_matmul_T_us": timed(lambda: torch.matmul(G, F.dequantize_4bit(qW, qs))),
                 "dequant_mm_bf16_to_fp32_us": timed(lambda: torch.mm(G, F.dequantize_4bit(qW, qs),
                                                                      out_dtype=torch.float32)),
                 "dequant_matmul_fp32_us": timed(lambda: torch.matmul(G.float(), F.dequantize_4bit(qW, qs).float()))}
            r["speedup_T"] = r["dequant_matmul_T_us"] / r["kernel_T_us"]
            r["speedup_fp32"] = r["dequant_mm_bf16_to_fp32_us"] / r["kernel_fp32_us"]
            rows.append(r)
            print(json.dumps(r), flush=True)
            del G, t_out, p_out
    res = {"gpu": gpu, "fp32_matmul_precision": torch.backends.cuda.matmul.fp32_precision, "reps": args.reps,
           "rows": rows}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "time_gemm4_input_grad.json").write_text(json.dumps(res, indent=1))
    print("gpu:", gpu)


if __name__ == "__main__":
    main()
