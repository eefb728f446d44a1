"""Time a data-parallel optimizer step of LoRA adapters eagerly and as a CUDA graph replay, alone and in a whole
QLoRA iteration:

  step: ShardedOptimizer.step() called from Python (per-piece config, launch arguments, grouping, ctypes calls);
  step graph: one replay of a CUDA graph that captured step() (capturable=True), collectives included;
  iteration: forward through Linear4bit bases plus the adapters, backward, clip_grad_norm_(1.0), step(), zero_grad();
  iteration graph: one replay of a CUDA graph that captured the whole iteration.

The adapters: rank 16 on every linear of Llama-3-8B's decoder layers (q, k, v, o, gate, up, down: 14 bf16 tensors per
layer, 448 for 32 layers); the frozen bases are NF4 Linear4bit layers of the same shapes.  Adam8bit and AdamW (32-bit
state).  The model is built once; the modes alternate for --rounds rounds in the same process, each run with a
fresh optimizer over it that warms up, then times --steps steps with CUDA events around each one (a step that leaves the GPU idle while
Python prepares launches shows that idle time).  The printed lines give the median of the round medians and their
range.  Run under ``python -m torch.distributed.run --nproc-per-node=W tools/time_sharded_graph.py --out DIR``; rank 0
writes DIR/time_sharded_graph_w{W}.json with the card's name and power limit, read in the same run.
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
from tools.time_sharded_optim import device_info, time_steps  # noqa: E402

_H, _KV, _FFN, _RANK = 4096, 1024, 14336, 16
_MAKERS = {"Adam8bit": lambda p: bnb.optim.Adam8bit(p, lr=1e-5, capturable=True),
           "AdamW": lambda p: bnb.optim.AdamW(p, lr=1e-5, capturable=True)}


class LoRA4bit(torch.nn.Module):
    """A frozen NF4 Linear4bit base plus trainable rank-16 adapters A [r, k] and B [n, r] (bf16)."""

    def __init__(self, k, n, dev, gen):
        super().__init__()
        self.base = bnb.nn.Linear4bit(k, n, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4", device="meta")
        w = torch.randn(n, k, generator=gen, device=dev, dtype=torch.bfloat16) / k**0.5
        self.base.weight = bnb.nn.Params4bit(w, requires_grad=False, quant_type="nf4", module=self.base).to(dev)
        self.A = torch.nn.Parameter(torch.randn(_RANK, k, generator=gen, device=dev, dtype=torch.bfloat16) / k**0.5)
        self.B = torch.nn.Parameter(torch.randn(n, _RANK, generator=gen, device=dev, dtype=torch.bfloat16) * 1e-3)

    def forward(self, x):
        return self.base(x) + (x @ self.A.t()) @ self.B.t()


class Layer(torch.nn.Module):
    """The seven projections of a decoder layer, without attention or norms: what the adapters see."""

    def __init__(self, dev, gen):
        super().__init__()
        self.q, self.o = LoRA4bit(_H, _H, dev, gen), LoRA4bit(_H, _H, dev, gen)
        self.k, self.v = LoRA4bit(_H, _KV, dev, gen), LoRA4bit(_H, _KV, dev, gen)
        self.gate, self.up = LoRA4bit(_H, _FFN, dev, gen), LoRA4bit(_H, _FFN, dev, gen)
        self.down = LoRA4bit(_FFN, _H, dev, gen)

    def forward(self, h):
        kv = torch.cat([self.k(h), self.v(h)], dim=-1).float().square().mean()
        h = h + self.o(self.q(h)) + self.down(torch.nn.functional.silu(self.gate(h)) * self.up(h))
        return h, kv


def build(layers, dev):
    """The model (built once: quantising the bases takes longer than the timed runs) and its adapters."""
    gen = torch.Generator(device=dev).manual_seed(0)
    model = torch.nn.ModuleList([Layer(dev, gen) for _ in range(layers)])
    return model, [p for n, p in model.named_parameters() if n.endswith((".A", ".B"))]


def run(mode, model, adapters, tokens, dev, warmup, steps, seed, kind):
    """Times of one mode with a fresh optimizer (each ShardedOptimizer moves the adapters into its own buffers)."""
    opt = bnb.optim.ShardedOptimizer(_MAKERS[kind](adapters))
    gen = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(tokens, _H, generator=gen, device=dev, dtype=torch.bfloat16)
    for p in adapters:
        p.grad.copy_(torch.randn(p.shape, generator=gen, device=dev, dtype=p.dtype) * 1e-3)

    def iteration():
        h, aux = x, 0.0
        for layer in model:
            h, kv = layer(h)
            aux = aux + kv
        (h.float().square().mean() + aux).backward()
        opt.clip_grad_norm_(1.0)
        opt.step()
        opt.zero_grad()

    body = opt.step if mode.startswith("step") else iteration
    if not mode.endswith("graph"):
        return time_steps(body, warmup, steps), len(adapters)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # the eager warm-up: state, buffers, NCCL's communicator
        for _ in range(max(1, warmup)):
            body()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    return time_steps(graph.replay, warmup, steps), len(adapters)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--tokens", type=int, default=512)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    result = {"world": world, "layers": args.layers, "tokens": args.tokens, "info": device_info(), "runs": []}
    modes = ["step", "step graph", "iteration", "iteration graph"]
    model, adapters = build(args.layers, dev)
    for kind in _MAKERS:
        rounds = {mode: [] for mode in modes}
        tensors = 0
        for _ in range(args.rounds):
            for mode in modes:
                t, tensors = run(mode, model, adapters, args.tokens, dev, args.warmup, args.steps, rank, kind)
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                dist.barrier()
                rounds[mode].append(t)
        for mode, ts in rounds.items():
            meds = [statistics.median(t) for t in ts]
            med = statistics.median(meds)
            result["runs"].append({"optimizer": kind, "tensors": tensors, "mode": mode, "median_ms": med,
                                   "round_medians_ms": meds, "samples_ms": ts})
            if rank == 0:
                print(f"w={world} {kind} {tensors} tensors, {args.layers} layers, {args.tokens} tokens, {mode}: "
                      f"{med:.3f} ms (round medians {min(meds):.3f} .. {max(meds):.3f}, {args.rounds} rounds x "
                      f"{args.steps} steps)", flush=True)
    if rank == 0:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"time_sharded_graph_w{world}.json"), "w") as f:
            json.dump(result, f, indent=1)
        print(json.dumps(result["info"]))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
