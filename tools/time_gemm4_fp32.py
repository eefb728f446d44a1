"""Times fp32 4-bit (NF4) GEMMs: the fp32 CUDA-core route against the TF32 tensor-core route, the dequantise + cuBLAS
route (under TF32 and under IEEE fp32), and the bf16 fused kernel for context.

For each weight shape N x K in {4096 x 4096, 11008 x 4096, 4096 x 11008} (blocksize 64, plain statistics) and each
token count M, every route is timed with CUDA events over --calls calls after a warm-up, --repeats times, the routes
alternating (the order reversed on every other repeat).  Routes:

    cuda_core   the library's fp32 route (native dtype 0: what fp32 takes under the default precision)
    tf32        the TF32 instance of the wgmma GEMM (native dtype 3 through the developer entry, so that it is timed
                below the dispatch threshold too)
    deq_tf32    dequantize_4bit(float32) + torch.matmul with fp32_precision = "tf32"  (cuBLAS)
    deq_ieee    the same with fp32_precision = "ieee"
    bf16        the bf16 fused GEMM on bf16 activations and weights, for context

Writes gemm4_fp32.json to --out with every sample, the medians and spreads, the device name, its power limit and
maximum SM clock, and for every timed size the agreement of the tf32 route with deq_tf32 (relative Frobenius norm of
the difference and the largest difference over the largest output).

    python tools/time_gemm4_fp32.py --out <dir>
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitsandbytes_b200.functional as F  # noqa: E402
from bitsandbytes_b200.cextension import lib  # noqa: E402

SHAPES = [(4096, 4096), (11008, 4096), (4096, 11008)]  # (N, K): output x input features
BS, NF4 = 64, 2


def device_info():
    info = {"device": torch.cuda.get_device_name(0), "torch": torch.__version__, "cuda": torch.version.cuda}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def stream():
    return torch.cuda.current_stream().cuda_stream


def native(x, q, absmax, out, N, K, dtype_id):
    M = x.shape[0]
    lib.cbnb_b200_gemm_4bit_strided(x.data_ptr(), q.data_ptr(), absmax.data_ptr(), None, None, None, out.data_ptr(),
                                    None, M, N, K, N, BS, NF4, dtype_id, stream())


def tf32_kernel(x, q, absmax, out, N, K):
    M = x.shape[0]
    rc = lib.cbnb_b200_gemm_4bit_pair(x.data_ptr(), q.data_ptr(), absmax.data_ptr(), None, None, None, out.data_ptr(),
                                      None, M, N, K, N, BS, NF4, 3, 0, 0, None, stream())
    if rc != 0:
        raise RuntimeError(f"the TF32 GEMM does not take M={M} N={N} K={K}")


def time_calls(fn, calls, precision):
    torch.backends.cuda.matmul.fp32_precision = precision
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e3 / calls  # microseconds per call


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory for gemm4_fp32.json")
    ap.add_argument("--tokens", type=int, nargs="+", default=[1, 2, 4, 8, 9, 16, 64, 256, 1024, 4096])
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_gemm4_fp32.py needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    prev = torch.backends.cuda.matmul.fp32_precision
    result = {"weights": f"NF4, blocksize {BS}, plain statistics", "calls": args.calls, "repeats": args.repeats,
              **device_info(), "rows": []}
    for N, K in SHAPES:
        g = torch.Generator(device="cpu").manual_seed(N + K)
        W = (torch.randn(N, K, generator=g) / K**0.5).cuda()
        q, st = F.quantize_4bit(W, blocksize=BS, quant_type="nf4", compress_statistics=False)
        W32 = F.dequantize_4bit(q, st)  # fp32
        q16, st16 = F.quantize_4bit(W.to(torch.bfloat16), blocksize=BS, quant_type="nf4", compress_statistics=False)
        for M in args.tokens:
            x = torch.randn(M, K, generator=g).cuda()
            x16 = x.to(torch.bfloat16)
            outs = {name: torch.empty(M, N, device="cuda") for name in ("cuda_core", "tf32")}
            out16 = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            routes = {
                "cuda_core": ("ieee", lambda: native(x, q, st.absmax, outs["cuda_core"], N, K, 0)),
                "tf32": ("ieee", lambda: tf32_kernel(x, q, st.absmax, outs["tf32"], N, K)),
                "deq_tf32": ("tf32", lambda: torch.matmul(x, F.dequantize_4bit(q, st).t())),
                "deq_ieee": ("ieee", lambda: torch.matmul(x, F.dequantize_4bit(q, st).t())),
                "bf16": ("ieee", lambda: native(x16, q16, st16.absmax, out16, N, K, 2)),
            }
            for prec, fn in routes.values():
                time_calls(fn, args.warmup, prec)
            lib.check("time_gemm4_fp32")
            torch.backends.cuda.matmul.fp32_precision = "tf32"
            ref = torch.matmul(x, W32.t())
            torch.backends.cuda.matmul.fp32_precision = "ieee"
            ref_ieee = torch.matmul(x, W32.t())
            torch.cuda.synchronize()
            agree = {}
            for name, ours in (("tf32", outs["tf32"]), ("cuda_core", outs["cuda_core"])):
                d = (ours.double() - ref.double())
                agree[name + "_vs_deq_tf32"] = {
                    "rel_fro": float(d.norm() / ref.double().norm()),
                    "max_over_max": float(d.abs().max() / ref.double().abs().max())}
            d = (ref.double() - ref_ieee.double())
            agree["deq_tf32_vs_deq_ieee"] = {"rel_fro": float(d.norm() / ref_ieee.double().norm()),
                                             "max_over_max": float(d.abs().max() / ref_ieee.double().abs().max())}
            samples = {name: [] for name in routes}
            names = list(routes)
            for r in range(args.repeats):
                for name in (names if r % 2 == 0 else names[::-1]):
                    samples[name].append(time_calls(routes[name][1], args.calls, routes[name][0]))
            lib.check("time_gemm4_fp32")
            row = {"N": N, "K": K, "M": M, "agreement": agree}
            for name, s in samples.items():
                row[name + "_us"] = statistics.median(s)
                row[name + "_spread_us"] = max(s) - min(s)
                row[name + "_samples_us"] = s
            row["tf32_speedup_vs_cuda_core"] = row["cuda_core_us"] / row["tf32_us"]
            row["tf32_speedup_vs_deq_tf32"] = row["deq_tf32_us"] / row["tf32_us"]
            row["tf32_tflops"] = 2.0 * M * N * K / row["tf32_us"] * 1e-6
            result["rows"].append(row)
            print(f"N={N:5d} K={K:5d} M={M:5d}  cuda_core {row['cuda_core_us']:9.1f}  tf32 {row['tf32_us']:8.1f}  "
                  f"deq_tf32 {row['deq_tf32_us']:8.1f}  deq_ieee {row['deq_ieee_us']:9.1f}  bf16 {row['bf16_us']:7.1f} us"
                  f"  x{row['tf32_speedup_vs_cuda_core']:.2f} vs cuda_core  "
                  f"rel_fro(tf32, deq_tf32) {agree['tf32_vs_deq_tf32']['rel_fro']:.2e}", flush=True)
        del W, q, W32, q16
    torch.backends.cuda.matmul.fp32_precision = prev
    with open(os.path.join(args.out, "gemm4_fp32.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(result["device"], "|", result["nvidia_smi"])


if __name__ == "__main__":
    main()
