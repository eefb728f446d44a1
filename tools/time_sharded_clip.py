"""Time gradient-norm clipping in a data-parallel optimizer step of AdamW8bit over bf16 parameters, three ways:

  step: ShardedOptimizer.step() without clipping;
  clip+step: ShardedOptimizer.clip_grad_norm_(1.0), then step() (the norm pass, one all-gather of one value per rank,
      the coefficient read by the update kernels on the device);
  replicated: all_reduce of a flat gradient buffer (the parameters' .grad are views of it, as DDP's buckets),
      torch.nn.utils.clip_grad_norm_(params, 1.0), then the multi-tensor step of the full optimizer on every rank.

It also times the norm launches alone (``optimizer_grad_norm_peers`` over this rank's pieces of every flat buffer) and
reports their achieved bytes/s, w x (this rank's elements) x sizeof(T) read per pass, against the H100 SXM data sheet's
3.35 TB/s.  Parameter lists: the linear and norm shapes of Llama-3-8B's decoder layers, for --layers counts.  The modes
alternate for --rounds rounds in the same process (each round builds its optimizer afresh, warms up, then times
--steps steps with CUDA events); the printed line gives the median of the round medians and their range.  Run under
``python -m torch.distributed.run --nproc-per-node=W tools/time_sharded_clip.py --out DIR``; rank 0 writes
DIR/time_sharded_clip_w{W}.json with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitsandbytes_b200 as bnb  # noqa: E402
from bitsandbytes_b200.backends.cuda import optimizer_grad_norm_peers  # noqa: E402
from tools.time_sharded_optim import device_info, fill_grads, llama3_8b_shapes, make_params, time_steps  # noqa: E402

_HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


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
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        opt.step()

    return time_steps(step, warmup, steps), None


def sharded(shapes, dev, warmup, steps, seed, clip):
    params = make_params(shapes, dev)
    opt = bnb.optim.ShardedOptimizer(bnb.optim.AdamW8bit(params, lr=1e-5))
    fill_grads(params, seed)

    def step():
        if clip:
            opt.clip_grad_norm_(1.0)
        opt.step()

    times = time_steps(step, warmup, steps)
    norm = None
    if clip:  # the norm launches alone, on the gradients as they are (no exchange: the local gradient as every source)
        acc = torch.zeros(1, dtype=torch.float64, device=dev)
        flats = [(f, [f.grad[s:s + n] for flat, _, s, n, _ in opt.pieces if flat is f]) for f in opt.flats]

        def launch():
            for f, pieces in flats:
                optimizer_grad_norm_peers(pieces, [f.grad.data_ptr()] * opt.world, f.grad, opt.grad_scale, 2.0, acc)

        elems = sum(n for *_, n, _ in opt.pieces)
        nbytes = opt.world * sum(n * f.grad.element_size() for f, _, _, n, _ in opt.pieces)
        launch()
        torch.cuda.synchronize()
        reps = 20
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            launch()
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b) / reps
        norm = {"elements": elems, "bytes": nbytes, "ms": ms, "bytes_per_s": nbytes / (ms * 1e-3),
                "share_of_3.35TB/s": nbytes / (ms * 1e-3) / _HBM_BYTES_PER_S}
    return times, norm


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
    modes = {"step": lambda *a: sharded(*a, clip=False), "clip+step": lambda *a: sharded(*a, clip=True),
             "replicated": replicated}
    for layers in args.layers:
        shapes = llama3_8b_shapes(layers)
        n = sum(torch.Size(s).numel() for s in shapes)
        rounds = {mode: [] for mode in modes}
        norms = []
        for _ in range(args.rounds):
            for mode, fn in modes.items():
                t, norm = fn(shapes, dev, args.warmup, args.steps, rank)
                torch.cuda.empty_cache()
                dist.barrier()
                rounds[mode].append(t)
                if norm is not None:
                    norms.append(norm)
        for mode, ts in rounds.items():
            meds = [statistics.median(t) for t in ts]
            med = statistics.median(meds)
            result["runs"].append({"layers": layers, "params": n, "mode": mode, "median_ms": med,
                                   "round_medians_ms": meds, "samples_ms": ts})
            if rank == 0:
                print(f"w={world} layers={layers} params={n / 1e9:.3f}B {mode}: {med:.2f} ms/step "
                      f"(round medians {min(meds):.2f} .. {max(meds):.2f}, {args.rounds} rounds x {args.steps} steps)",
                      flush=True)
        ms = [q["ms"] for q in norms]
        norm = dict(norms[0], ms=statistics.median(ms), round_ms=ms)
        norm["bytes_per_s"] = norm["bytes"] / (norm["ms"] * 1e-3)
        norm["share_of_3.35TB/s"] = norm["bytes_per_s"] / _HBM_BYTES_PER_S
        result["runs"].append({"layers": layers, "params": n, "mode": "norm launches", **norm})
        if rank == 0:
            print(f"w={world} layers={layers} norm launches: {norm['ms']:.3f} ms for {norm['bytes'] / 1e9:.2f} GB, "
                  f"{norm['bytes_per_s'] / 1e12:.2f} TB/s ({100 * norm['share_of_3.35TB/s']:.0f} % of 3.35 TB/s; "
                  f"rounds {min(ms):.3f} .. {max(ms):.3f} ms)", flush=True)
    if rank == 0:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"time_sharded_clip_w{world}.json"), "w") as f:
            json.dump(result, f, indent=1)
        print(json.dumps(result["info"]))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
