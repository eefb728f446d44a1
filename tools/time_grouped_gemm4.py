#!/usr/bin/env python
"""Timings of the grouped 4-bit GEMM against the other ways to run a mixture-of-experts layer on 4-bit experts
(CUDA events, one GPU).

    python tools/time_grouped_gemm4.py --out DIR [--reps 20]

Shapes (NF4, blocksize 64, plain statistics, bf16): Mixtral-8x7B gate_up [8, 28672, 4096] and down [8, 4096, 14336]
with top-2 routing, Qwen3-30B-A3B gate_up [128, 1536, 2048] and down [128, 2048, 768] with top-8 routing; 1, 16, 256
and 4096 tokens, routed by a seeded top-k of uniform router scores.  Routes:

* ``grouped``: gemm_4bit_grouped at the production token tile, and ``grouped_mt<T>`` at each tile T;
* ``dequant_all+grouped_mm``: dequantise the whole expert tensor, then torch.nn.functional.grouped_mm (what the
  parametrize route costs per forward);
* ``per_expert_loop``: the expert counts read to the host (a synchronisation), then one bnb.matmul_4bit per routed
  expert;
* ``grouped_mm_16bit``: grouped_mm on already dequantised bf16 weights (the 16-bit reference point).

Per shape, the FLOPs (2 x rows x N x K) and the bytes the grouped kernel must move (the routed experts' codes and
scales, the activations and the output) are computed from the shapes; ``share`` is the larger of FLOPs / 989 TFLOP/s
and bytes / 3.35 TB/s (the H100 SXM data sheet's dense bf16 rate and HBM3 bandwidth) over the measured time, with the
bound that applies.  Writes DIR/time_grouped_gemm4.json and prints one JSON line per measurement, with the card's name
and power limit read in the same run.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SHAPES = (("mixtral_gate_up", 8, 28672, 4096, 2), ("mixtral_down", 8, 4096, 14336, 2),
          ("qwen3_gate_up", 128, 1536, 2048, 8), ("qwen3_down", 128, 2048, 768, 8))
TOKENS = (1, 16, 256, 4096)
MTS = (16, 32, 64, 128)
PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()

    import torch

    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F
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
    print(json.dumps({"gpu": gpu}), flush=True)
    rows = []
    for name, E, N, K, topk in SHAPES:
        torch.manual_seed(0)
        W = (torch.randn(E, N, K, device=dev) / K**0.5).to(torch.bfloat16)
        qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="nf4")
        Wd = F.dequantize_4bit(qW, qs)  # [E, N, K] bf16, the 16-bit reference's weights
        del W
        per = N * K
        per_expert = [(qW.view(-1)[e * per // 2:(e + 1) * per // 2].view(-1, 1),
                       F.QuantState(absmax=qs.absmax[e * per // 64:(e + 1) * per // 64], shape=torch.Size([N, K]),
                                    code=qs.code, blocksize=64, quant_type="nf4", dtype=torch.bfloat16))
                      for e in range(E)]
        for T in TOKENS:
            g = torch.Generator().manual_seed(T)
            choice = torch.rand(T, E, generator=g).topk(topk, dim=1).indices.reshape(-1)
            counts = torch.bincount(choice, minlength=E)
            M = T * topk
            offs = counts.cumsum(0).to(torch.int32).to(dev)
            x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
            active = int((counts > 0).sum())
            flops = 2.0 * M * N * K
            nbytes = active * (per // 2 + per // 64 * 4) + M * K * 2 + M * N * 2
            bound = max(flops / PEAK_FLOPS, nbytes / PEAK_BYTES) * 1e6
            bound_by = "compute" if flops / PEAK_FLOPS > nbytes / PEAK_BYTES else "memory"

            out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)

            def grouped_mt(mt):
                return lambda: lib.cbnb_b200_gemm_4bit_grouped_mt(
                    x.data_ptr(), qW.data_ptr(), qs.absmax.data_ptr(), None, None, None, offs.data_ptr(), E,
                    out.data_ptr(), None, M, N, K, N, 64, 2, 2, mt, torch.cuda.current_stream().cuda_stream)

            def dequant_all():
                Wt = F.dequantize_4bit(qW, qs)
                return torch.nn.functional.grouped_mm(x, Wt.transpose(1, 2), offs=offs)

            def per_expert_loop():
                s = 0
                for e, t in enumerate(offs.cpu().tolist()):  # the host read of the routing
                    if t > s:
                        bnb.matmul_4bit(x[s:t], per_expert[e][0], per_expert[e][1])
                    s = t

            routes = {"grouped": lambda: bnb.grouped_matmul_4bit(x, qW, qs, offs)}
            for mt in MTS:
                routes[f"grouped_mt{mt}"] = grouped_mt(mt)
            routes["dequant_all+grouped_mm"] = dequant_all
            routes["per_expert_loop"] = per_expert_loop
            routes["grouped_mm_16bit"] = lambda: torch.nn.functional.grouped_mm(x, Wd.transpose(1, 2), offs=offs)
            mean = -(M // -E)
            for route, fn in routes.items():
                us = timed(fn)
                r = {"shape": name, "E": E, "N": N, "K": K, "tokens": T, "rows": M, "mean_rows": mean,
                     "active_experts": active, "route": route, "us": round(us, 2), "flops": flops, "bytes": nbytes,
                     "bound_us": round(bound, 2), "bound_by": bound_by, "share": round(bound / us, 3)}
                rows.append(r)
                print(json.dumps(r), flush=True)
        del Wd, qW, per_expert
        torch.cuda.empty_cache()
    d = Path(args.out)
    d.mkdir(parents=True, exist_ok=True)
    (d / "time_grouped_gemm4.json").write_text(json.dumps({"gpu": gpu, "reps": args.reps, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
