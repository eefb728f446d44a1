"""Times optimizer.step() eager against the replay of a CUDA graph that captured one step() (capturable=True), on the
sets of tools/time_optim_step.py (the LoRA set of a Llama-3-8B at r = 16 and r = 64, 448 bf16 tensors, and the
large-tensor set), for AdamW8bit, AdamW (32-bit state) and Lion8bit.  Routes:

* eager: the grouped step with capturable=False (the default);
* eager_capturable: the same step with capturable=True (device step counters: one more, tiny, kernel per launch);
* graph: torch.cuda.CUDAGraph.replay() of one captured step() of a capturable optimizer.

Per route, --repeats samples of --steps steps after --warmup eager steps, the routes alternating (and swapping which
goes first): host time = a wall clock around the steps that ends in torch.cuda.synchronize(); event time = CUDA events
around the same steps.  Every route starts from the same parameters and runs the same number of steps on the same
(fixed) gradients, so their parameters must end bit-identical; the JSON records it.

Also one whole QLoRA layer step, eager (AdamW8bit, capturable=False) against the replay of a graph that captured it
(capturable=True): an NF4 Linear4bit base (4096 x 4096, bf16 compute, frozen) with LoRA A / B (r = 16), 2048 tokens,
forward, MSE loss, backward and step().  Writes optim_graph.json to --out with every sample, the medians, the device
name and its power limit.

    python tools/time_optim_graph.py --out <dir>
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_optim_step import SETS, device_info, make_params  # noqa: E402

import bitsandbytes_b200 as bnb  # noqa: E402

OPTIMIZERS = {
    "AdamW8bit": lambda ps, cap: bnb.optim.AdamW8bit(ps, lr=1e-4, capturable=cap),
    "AdamW32bit": lambda ps, cap: bnb.optim.AdamW(ps, lr=1e-4, capturable=cap),
    "Lion8bit": lambda ps, cap: bnb.optim.Lion8bit(ps, lr=1e-5, capturable=cap),
}


def time_calls(fn, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3, start.elapsed_time(end) / steps


def capture(fn):
    """The graph of one fn() call, captured after the caller's eager warm-up."""
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


def alternate(routes, args):
    """{route: callable}: samples of args.steps calls per route, alternating; returns the samples and medians."""
    samples = {k: {"host_ms": [], "event_ms": []} for k in routes}
    order = list(routes)
    for r in range(args.repeats):
        for k in (order if r % 2 == 0 else order[::-1]):
            h, e = time_calls(routes[k], args.steps)
            samples[k]["host_ms"].append(h)
            samples[k]["event_ms"].append(e)
    return {k: {"host_ms_median": statistics.median(v["host_ms"]), "event_ms_median": statistics.median(v["event_ms"]),
                **v} for k, v in samples.items()}


def bitwise(a, b):
    return all(torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(a, b))


def run_set(set_name, args):
    shapes = SETS[set_name]()
    res = {"tensors": len(shapes), "elements": sum(a * b for a, b in shapes), "optimizers": {}}
    for oname, make in OPTIMIZERS.items():
        params = {k: make_params(shapes) for k in ("eager", "eager_capturable", "graph")}
        opts = {"eager": make(params["eager"], False), "eager_capturable": make(params["eager_capturable"], True),
                "graph": make(params["graph"], True)}
        for o in opts.values():
            for _ in range(args.warmup):
                o.step()
        graph = capture(opts["graph"].step)
        out = alternate({"eager": opts["eager"].step, "eager_capturable": opts["eager_capturable"].step,
                         "graph": graph.replay}, args)
        out["routes_bitwise_equal"] = (bitwise(params["eager"], params["eager_capturable"])
                                       and bitwise(params["eager"], params["graph"]))
        out["speedup_host_graph_vs_eager"] = out["eager"]["host_ms_median"] / out["graph"]["host_ms_median"]
        res["optimizers"][oname] = out
        line = "  ".join(f"{k} {out[k]['host_ms_median']:.3f} ms host / {out[k]['event_ms_median']:.3f} ms events"
                         for k in opts)
        print(f"{set_name:9s} {oname:11s} {line}  bitwise={out['routes_bitwise_equal']}  "
              f"x{out['speedup_host_graph_vs_eager']:.2f}", flush=True)
        del opts, params, graph
        torch.cuda.empty_cache()
    return res


class LoRALinear4bit(torch.nn.Module):
    def __init__(self, k, n, r, seed):
        super().__init__()
        g = torch.Generator(device="cpu").manual_seed(seed)
        lin = torch.nn.Linear(k, n, bias=False)
        with torch.no_grad():
            lin.weight.copy_(torch.randn(n, k, generator=g) / k**0.5)
        self.base = bnb.nn.Linear4bit(k, n, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4")
        self.base.load_state_dict(lin.state_dict())
        self.base = self.base.cuda()
        self.A = torch.nn.Parameter((torch.randn(r, k, generator=g) / k**0.5).to(torch.bfloat16).cuda())
        self.B = torch.nn.Parameter((torch.randn(n, r, generator=g) * 0.01).to(torch.bfloat16).cuda())

    def forward(self, x):
        return self.base(x) + (x @ self.A.t()) @ self.B.t()


def run_qlora(args, k=4096, n=4096, r=16, tokens=2048):
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(tokens, k, device="cuda", generator=g, dtype=torch.bfloat16)
    y = torch.randn(tokens, n, device="cuda", generator=g, dtype=torch.bfloat16)
    layers = {cap: LoRALinear4bit(k, n, r, seed=0) for cap in (False, True)}
    opts = {cap: bnb.optim.AdamW8bit([m.A, m.B], lr=1e-4, capturable=cap) for cap, m in layers.items()}

    def step(cap):
        opts[cap].zero_grad(set_to_none=not cap)  # (the graph's .grad tensors stay; eager steps set them anew)
        torch.nn.functional.mse_loss(layers[cap](x), y).backward()
        opts[cap].step()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(args.warmup):
            step(False)
            step(True)
    torch.cuda.current_stream().wait_stream(side)
    opts[True].zero_grad(set_to_none=True)
    graph = capture(lambda: step(True))
    out = alternate({"eager": lambda: step(False), "graph": graph.replay}, args)
    pa, pb = [layers[False].A, layers[False].B], [layers[True].A, layers[True].B]
    out["routes_bitwise_equal"] = bitwise(pa, pb)
    out["max_abs_param_diff"] = max(float((a.detach().float() - b.detach().float()).abs().max()) for a, b in zip(pa, pb))
    out["speedup_host_graph_vs_eager"] = out["eager"]["host_ms_median"] / out["graph"]["host_ms_median"]
    print(f"qlora     eager {out['eager']['host_ms_median']:.3f} ms host / {out['eager']['event_ms_median']:.3f} ms "
          f"events  graph {out['graph']['host_ms_median']:.3f} / {out['graph']['event_ms_median']:.3f} ms  "
          f"bitwise={out['routes_bitwise_equal']}  x{out['speedup_host_graph_vs_eager']:.2f}", flush=True)
    return {"k": k, "n": n, "r": r, "tokens": tokens, **out}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for optim_graph.json")
    ap.add_argument("--sets", default=",".join(SETS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_optim_graph.py needs a CUDA device")
    info = device_info()
    print(info, flush=True)
    result = {"info": info, "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "sets": {}}
    for s in args.sets.split(","):
        result["sets"][s] = run_set(s, args)
    result["qlora_layer"] = run_qlora(args)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "optim_graph.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
