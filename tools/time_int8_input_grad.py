#!/usr/bin/env python
"""Timings of the input-gradient path of the tensor-parallel LLM.int8() layers (CUDA events, one GPU).

    python tools/time_int8_input_grad.py --out DIR [--reps 50]

Shards of a Llama-70B MLP at tensor-parallel world 8, bf16: the column shard of the up projection (8192 -> 28672/8,
weight 3584 x 8192) and the row shard of the down projection (28672/8 -> 8192, weight 8192 x 3584).  For each weight:
  * the one-pass dequantisation (int8_dequant_rows) against the torch expression of MatMul8bitLt.backward,
    CB.to(T).mul_(SCB.unsqueeze(1).mul(1/127)), in us and in GB/s against the bytes each needs (3 N K for one pass that
    reads the codes once and writes T once, 7 N K for the two passes with their temporary);
  * the layer's per-rank backward (``_backward`` at world 1: the dequantisation, the cuBLAS product -- fp32 partial and
    reduce_partials for the column layer, the rounded product for the row layer -- without the exchange) at M in
    {256, 2048, 4096}, and the share of the dequantisation in it.
Writes DIR/time_int8_input_grad.json, with the card's name and power limit read in the same run, and prints one line
per measurement.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SHARDS = (("column", 3584, 8192, 28672), ("row", 8192, 3584, 28672))  # (layer, N rows of the shard, K, full width)
MS = (256, 2048, 4096)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()

    import torch

    from bitsandbytes_b200.backends.cuda import int8_dequant_rows
    from bitsandbytes_b200.cextension import lib
    from bitsandbytes_b200.parallel import ColumnParallelLinear8bitLt, RowParallelLinear8bitLt, Shard8bit

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")
    dtype = torch.bfloat16

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
    for kind, N, K, width in SHARDS:
        g = torch.Generator(device=dev).manual_seed(N)
        CB = torch.randint(-127, 128, (N, K), device=dev, dtype=torch.int8, generator=g)
        SCB = torch.rand(N, device=dev, generator=g) * 0.1 + 0.01
        out = torch.empty(N, K, device=dev, dtype=dtype)
        want = CB.to(dtype, copy=True).mul_(SCB.unsqueeze(1).mul(1.0 / 127.0))
        assert torch.equal(int8_dequant_rows(CB, SCB, dtype, out=out).view(torch.int16), want.view(torch.int16))
        one = timed(lambda: int8_dequant_rows(CB, SCB, dtype, out=out))
        two = timed(lambda: CB.to(dtype, copy=True).mul_(SCB.unsqueeze(1).mul(1.0 / 127.0)))
        r = {"what": "dequant", "layer": kind, "N": N, "K": K, "dequant_rows_us": one, "torch_expression_us": two,
             "dequant_rows_GBps": 3 * N * K / one / 1e3, "torch_expression_GBps": 7 * N * K / two / 1e3,
             "speedup": two / one}
        rows.append(r)
        print(json.dumps(r), flush=True)
        if kind == "column":
            layer = ColumnParallelLinear8bitLt(Shard8bit(CB=CB, SCB=SCB, rows=N, row0=0, K=K), width,
                                               gather_output=False)
        else:
            layer = RowParallelLinear8bitLt(Shard8bit(CB=CB, SCB=SCB, rows=N, row0=0, K=K), width)
        for M in MS:
            gy = torch.randn(M, N, device=dev, generator=g).to(dtype)
            bwd = timed(lambda: layer._backward(gy, (M, K)))
            r = {"what": "backward", "layer": kind, "N": N, "K": K, "M": M, "backward_us": bwd,
                 "dequant_share": one / bwd}
            rows.append(r)
            print(json.dumps(r), flush=True)
            del gy
        del CB, SCB, out, want, layer
    res = {"gpu": gpu, "reps": args.reps, "dtype": "bf16", "rows": rows}
    out_dir = Path(args.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    (out_dir / "time_int8_input_grad.json").write_text(json.dumps(res, indent=1))
    print("gpu:", gpu)


if __name__ == "__main__":
    main()
