#!/usr/bin/env python
"""Time the backward of the tensor-parallel Linear4bit layers through the symmetric-memory exchange (the fused routes
with ``grad_peers``) against the NCCL exchange (the layers' own forward), on every GPU of the machine.

    python tools/time_parallel_backward_fused.py --out DIR [--reps 20] [--repeats 3]

Launches one process per visible GPU (``torch.distributed.run``) unless it already runs under it.  For each route
family -- column (gathered output), column with sequence parallelism, row with the whole input
(``input_is_parallel=False``), row with sequence parallelism, and the plain row layer, which exchanges nothing -- at
M in {256, 2048, 4096} tokens on a 4096 x 4096 weight and on 11008 x 4096 (column) / 4096 x 11008 (row) weights
(shapes that do not shard over the world are left out): one forward with an input that requires grad, then
``torch.autograd.grad`` of that output, timed with CUDA events over ``--reps`` calls after 3 warm-up calls, the NCCL
and the fused backward alternated ``--repeats`` times.  NF4, bf16; the int8 layers share this backward.  Rank 0
writes DIR/time_parallel_backward_fused.json with the card's name and power limit, read in the same run, and prints
one line per measurement.  For the gathered column route it also times the inference forward and the copy of the
``[M, N]`` output slot that a training call adds.  With one GPU the exchange is empty: the numbers are each route's
own overhead.
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

MS = (256, 2048, 4096)
SHAPES = ((4096, 4096), (11008, 4096))  # column weight [N, K]; the row layer takes its transpose [K, N]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import torch

    if "RANK" not in os.environ:
        n = torch.cuda.device_count()
        if n == 0:
            raise SystemExit("needs a CUDA device")
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
                            "--master-addr", "127.0.0.1", "--master-port", "29711", __file__] + sys.argv[1:])
        raise SystemExit(r.returncode)

    import torch.distributed as dist

    import bitsandbytes_b200.functional as F
    import bitsandbytes_b200.parallel as par
    from bitsandbytes_b200.cextension import lib

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    dt = torch.bfloat16

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        dist.barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        lib.check("timed call")
        return a.elapsed_time(b) * 1e3 / args.reps  # us per backward

    def weights(N, K, seed):
        torch.manual_seed(seed)
        return F.quantize_4bit((torch.randn(N, K, device=dev) / K**0.5).to(dt), quant_type="nf4")

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    rows = []
    for N, K in SHAPES:
        cq, cs = weights(N, K, 1)   # column: K -> N
        rq, rs = weights(K, N, 2)   # row: N -> K
        for M in MS:
            if N % world or M % world or N % (world * 64):
                continue
            Ms = M // world
            col = par.ColumnParallelLinear4bit.from_quantized(cq, cs)
            col_sp = par.ColumnParallelLinear4bit.from_quantized(cq, cs, gather_output=False, sequence_parallel=True)
            row = par.RowParallelLinear4bit.from_quantized(rq, rs)
            row_full = par.RowParallelLinear4bit.from_quantized(rq, rs, input_is_parallel=False)
            row_sp = par.RowParallelLinear4bit.from_quantized(rq, rs, sequence_parallel=True)
            x = torch.randn(M, K, device=dev, dtype=dt)
            h = torch.randn(M, N, device=dev, dtype=dt)
            h_r = h[:, rank * N // world:(rank + 1) * N // world].contiguous()
            g_col = par.PeerInputGrad(M, K, torch.float32, dev)
            cases = [("column", col, x, par.fused_forward, (par.PeerGather(M, N, dt, dev), g_col)),
                     ("column SP", col_sp, x[rank * Ms:(rank + 1) * Ms].contiguous(), par.fused_forward_col_sp,
                      (par.PeerGather(M, K, dt, dev), g_col)),
                     ("row, whole input", row_full, h, par.fused_forward_row,
                      (par.PeerPartials(M, K, dev), par.PeerInputGrad(M, N, dt, dev))),
                     ("row SP", row_sp, h_r, par.fused_forward_row_sp,
                      (par.PeerPartials(Ms, K, dev), par.PeerInputGrad(M, K, dt, dev))),
                     ("row", row, h_r, par.fused_forward_row,
                      (par.PeerPartials(M, K, dev), par.PeerInputGrad(M, N, dt, dev)))]
            for family, layer, inp, route, peers in cases:
                xa = inp.detach().clone().requires_grad_()
                ya = route(layer, xa, *peers)
                xb = inp.detach().clone().requires_grad_()
                yb = layer(xb)
                gy = torch.randn(ya.shape, device=dev, dtype=dt)
                ga = torch.autograd.grad(ya, xa, gy, retain_graph=True)[0]
                gb = torch.autograd.grad(yb, xb, gy, retain_graph=True)[0]
                assert torch.equal(ga, gb), f"{family}: the fused gradient differs from the NCCL one"
                nccl, fused = [], []
                for _ in range(args.repeats):
                    nccl.append(timed(lambda: torch.autograd.grad(yb, xb, gy, retain_graph=True)))
                    fused.append(timed(lambda: torch.autograd.grad(ya, xa, gy, retain_graph=True)))
                rec = dict(family=family, weight=f"{N}x{K}" if family.startswith("column") else f"{K}x{N}", M=M,
                           world=world, nccl_us=sorted(round(t, 1) for t in nccl),
                           fused_us=sorted(round(t, 1) for t in fused))
                if family == "column":
                    # the gathered column route returns its output slot; a training call returns a copy of it
                    with torch.no_grad():
                        rec["forward_us"] = round(timed(lambda: route(layer, inp, peers[0])), 1)
                    rec["output_copy_us"] = round(timed(lambda: ya.clone()), 1)
                rows.append(rec)
                if rank == 0:
                    print(json.dumps(rec), flush=True)
            del col, col_sp, row, row_full, row_sp
            torch.cuda.empty_cache()
    if rank == 0:
        out = Path(args.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / "time_parallel_backward_fused.json").write_text(json.dumps(dict(gpu=gpu, world=world, reps=args.reps,
                                                                               rows=rows), indent=1))
        print(json.dumps(dict(gpu=gpu, world=world)))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
