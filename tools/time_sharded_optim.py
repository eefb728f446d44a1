"""Time one data-parallel optimizer step of AdamW8bit over bf16 parameters, two ways, per rank count:

  replicated: all_reduce of a flat gradient buffer (the parameters' .grad are views of it, as DDP's buckets), then
      the multi-tensor step of the full optimizer on every rank;
  sharded: ShardedOptimizer: all_to_all_single of the gradient, the rank's pieces updated by the peer kernel,
      all_gather_into_tensor of the parameters (with one rank: the peer kernel alone).

Parameter lists: the linear and norm shapes of Llama-3-8B's decoder layers (q, k, v, o, gate, up, down, two RMSNorm
weights per layer), for --layers counts.  The two modes alternate for --rounds rounds in the same process (each round
builds its optimizer afresh, warms up, then times --steps steps with CUDA events); the JSON keeps every sample, and the
printed line gives the median of the round medians and their range.  Run under
``python -m torch.distributed.run --nproc-per-node=W tools/time_sharded_optim.py --out DIR``; rank 0 writes
DIR/time_sharded_optim_w{W}.json with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitsandbytes_b200 as bnb  # noqa: E402


def device_info():
    info = {"device": torch.cuda.get_device_name(), "torch": torch.__version__, "cuda": torch.version.cuda}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}",
                            "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def llama3_8b_shapes(layers):
    h, kv, ffn = 4096, 1024, 14336
    per = [(h, h), (kv, h), (kv, h), (h, h), (ffn, h), (ffn, h), (h, ffn), (h,), (h,)]
    return per * layers


def make_params(shapes, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    return [torch.nn.Parameter(torch.randn(s, generator=g, device=dev, dtype=torch.bfloat16) * 0.02) for s in shapes]


def fill_grads(params, seed):
    g = torch.Generator(device=params[0].device).manual_seed(seed)
    for p in params:
        p.grad.copy_(torch.randn(p.shape, generator=g, device=p.device, dtype=p.dtype) * 1e-3)


def time_steps(step, warmup, steps):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    dist.barrier()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return times


def replicated(shapes, dev, warmup, steps, seed):
    params = make_params(shapes, dev)
    flat = torch.zeros(sum(p.numel() for p in params), dtype=torch.bfloat16, device=dev)
    o = 0
    for p in params:
        p.grad = flat[o:o + p.numel()].view_as(p)
        o += p.numel()
    fill_grads(params, seed)
    opt = bnb.optim.AdamW8bit(params, lr=1e-5)

    def step():
        dist.all_reduce(flat)
        opt.step()

    return time_steps(step, warmup, steps)


def sharded(shapes, dev, warmup, steps, seed):
    params = make_params(shapes, dev)
    opt = bnb.optim.ShardedOptimizer(bnb.optim.AdamW8bit(params, lr=1e-5))
    fill_grads(params, seed)
    return time_steps(opt.step, warmup, steps)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--layers", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    result = {"world": world, "info": device_info(), "runs": []}
    for layers in args.layers:
        shapes = llama3_8b_shapes(layers)
        n = sum(torch.Size(s).numel() for s in shapes)
        rounds = {"replicated": [], "sharded": []}
        for _ in range(args.rounds):
            for mode in rounds:
                fn = replicated if mode == "replicated" else sharded
                t = fn(shapes, dev, args.warmup, args.steps, rank)
                torch.cuda.empty_cache()
                dist.barrier()
                rounds[mode].append(t)
        for mode, ts in rounds.items():
            meds = [statistics.median(t) for t in ts]
            med = statistics.median(meds)
            result["runs"].append({"layers": layers, "params": n, "mode": mode, "median_ms": med,
                                   "round_medians_ms": meds, "samples_ms": ts})
            if rank == 0:
                print(f"w={world} layers={layers} params={n / 1e9:.3f}B {mode}: {med:.2f} ms/step "
                      f"(round medians {min(meds):.2f} .. {max(meds):.2f}, {args.rounds} rounds x {args.steps} steps)",
                      flush=True)
    if rank == 0:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"time_sharded_optim_w{world}.json"), "w") as f:
            json.dump(result, f, indent=1)
        print(json.dumps(result["info"]))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
