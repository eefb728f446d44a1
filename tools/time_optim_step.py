"""Times optimizer.step() of the 8-bit / 32-bit optimizers with the grouped multi-tensor step against the per-parameter
loop the optimizers ran before it (one F.optimizer_update_* call per parameter, restated below), on

* the LoRA set of a Llama-3-8B: A / B on all seven projections of the 32 layers, r = 16 and r = 64, bf16 (448 tensors);
* a full-finetune-like set of large tensors (4 x 4096x4096 + 2 x 14336x4096, bf16), where the update is bound by HBM.

Optimizers: AdamW8bit, PagedAdamW8bit, AdamW (32-bit state), Lion8bit, and torch.optim.AdamW(fused=True) for context.
Per route, --repeats samples of --steps steps after --warmup steps, the routes alternating (and swapping which goes
first): host time = a wall clock around the steps that ends in torch.cuda.synchronize(); event time = CUDA events
around the same steps.  After the timed steps, one more step per route of every optimizer but the paged one runs
under torch.profiler (CUDA activities, one session per set) for the kernel count and the summed kernel time.  Both
routes start from the same parameters and run the same steps on the same gradients, so their parameters must end
bit-identical; the JSON records it.  Writes optim_step.json to --out with every sample, the
medians, the device name and its power limit.

    python tools/time_optim_step.py --out <dir>
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitsandbytes_b200 as bnb  # noqa: E402
import bitsandbytes_b200.functional as F  # noqa: E402


def device_info():
    info = {"device": torch.cuda.get_device_name(0), "torch": torch.__version__, "cuda": torch.version.cuda}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def lora_shapes(r):
    proj = [(4096, 4096), (4096, 1024), (4096, 1024), (4096, 4096), (4096, 14336), (4096, 14336), (14336, 4096)]
    return [s for _ in range(32) for i, o in proj for s in ((r, i), (o, r))]


SETS = {
    "lora_r16": lambda: lora_shapes(16),
    "lora_r64": lambda: lora_shapes(64),
    "full": lambda: [(4096, 4096)] * 4 + [(14336, 4096)] * 2,
}


def per_parameter(cls):
    """The optimizer with the per-parameter update_step of the library before the multi-tensor step (one
    F.optimizer_update_* call per parameter)."""

    class PerParameter(cls):
        @torch.no_grad()
        def update_step(self, group, p, gindex, pindex):
            p.data = p.data.contiguous()
            p.grad = p.grad.contiguous()
            state = self.state[p]
            config = self.get_config(gindex, pindex, group)
            state["step"] += 1
            beta1, beta2 = config["betas"][0], config["betas"][1]
            two = "state2" in state
            if state["state1"].dtype == torch.float32:
                F.optimizer_update_32bit(self.optimizer_name, p.grad, p, state["state1"], beta1, config["eps"],
                                         state["step"], config["lr"], state["state2"] if two else None, beta2, 0.0, 0.0,
                                         config["weight_decay"], 1.0, None, max_unorm=0.0,
                                         skip_zeros=config["skip_zeros"])
            else:
                F.optimizer_update_8bit_blockwise(self.optimizer_name, p.grad, p, state["state1"],
                                                  state["state2"] if two else None, beta1, beta2, 0.0, 0.0,
                                                  config["eps"], state["step"], config["lr"], state["qmap1"],
                                                  state["qmap2"] if two else None, state["absmax1"],
                                                  state["absmax2"] if two else None, config["weight_decay"],
                                                  gnorm_scale=1.0, skip_zeros=config["skip_zeros"])

    return PerParameter


OPTIMIZERS = {
    "AdamW8bit": lambda ps, per: (per_parameter(bnb.optim.AdamW8bit) if per else bnb.optim.AdamW8bit)(ps, lr=1e-4),
    "PagedAdamW8bit": lambda ps, per: (per_parameter(bnb.optim.PagedAdamW8bit) if per else bnb.optim.PagedAdamW8bit)(
        ps, lr=1e-4),
    "AdamW32bit": lambda ps, per: (per_parameter(bnb.optim.AdamW) if per else bnb.optim.AdamW)(ps, lr=1e-4),
    "Lion8bit": lambda ps, per: (per_parameter(bnb.optim.Lion8bit) if per else bnb.optim.Lion8bit)(ps, lr=1e-5),
}


def make_params(shapes, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ps = []
    for s in shapes:
        p = torch.nn.Parameter(torch.randn(s, device="cuda", generator=g, dtype=torch.bfloat16) * 0.02)
        p.grad = torch.randn(s, device="cuda", generator=g, dtype=torch.bfloat16) * 1e-3
        ps.append(p)
    return ps


def time_steps(opt, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    start.record()
    for _ in range(steps):
        opt.step()
    end.record()
    torch.cuda.synchronize()
    host = (time.perf_counter() - t0) / steps
    return host * 1e3, start.elapsed_time(end) / steps


def profile_steps(routes):
    """One step per route in one profiler session, each inside a named range that ends in a synchronise: the kernels
    that start inside a route's range are its kernels.  Returns {route: (kernels, summed kernel time in ms)}."""
    from torch.profiler import ProfilerActivity, profile, record_function

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)  # (the first kernels of a session can go unrecorded)
        torch.cuda.synchronize()
        for k, o in routes.items():
            with record_function(f"route:{k}"):
                o.step()
                torch.cuda.synchronize()
    events = prof.events()
    ranges = {e.name[len("route:"):]: e.time_range for e in events if e.name.startswith("route:")}
    kernels = [e for e in events if e.device_type == torch.autograd.DeviceType.CUDA and e.name.startswith("void")]
    out = {}
    for k, r in ranges.items():
        mine = [e for e in kernels if r.start <= e.time_range.start <= r.end]
        out[k] = (len(mine), sum(e.device_time for e in mine) / 1e3)
    return out


def run_set(set_name, args):
    shapes = SETS[set_name]()
    numel = sum(a * b for a, b in shapes)
    res = {"tensors": len(shapes), "elements": numel, "optimizers": {}}
    kept = {}  # every optimizer's routes, profiled together at the end of the set
    for oname, make in OPTIMIZERS.items():
        routes = {"grouped": make(make_params(shapes), False), "per_parameter": make(make_params(shapes), True)}
        params = {k: [p for grp in o.param_groups for p in grp["params"]] for k, o in routes.items()}
        if oname == "AdamW8bit":
            routes["torch_fused_AdamW"] = torch.optim.AdamW(make_params(shapes), lr=1e-4, fused=True)
        samples = {k: {"host_ms": [], "event_ms": []} for k in routes}
        for o in routes.values():
            for _ in range(args.warmup):
                o.step()
        order = list(routes)
        for r in range(args.repeats):
            for k in (order if r % 2 == 0 else order[::-1]):
                h, e = time_steps(routes[k], args.steps)
                samples[k]["host_ms"].append(h)
                samples[k]["event_ms"].append(e)
        out = {k: {"host_ms_median": statistics.median(v["host_ms"]), "event_ms_median": statistics.median(v["event_ms"]),
                   **v} for k, v in samples.items()}
        # both routes ran warmup + repeats * steps steps on the same gradients
        out["grouped_equals_per_parameter_bitwise"] = all(
            torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(params["grouped"], params["per_parameter"]))
        out["speedup_host"] = out["per_parameter"]["host_ms_median"] / out["grouped"]["host_ms_median"]
        res["optimizers"][oname] = out
        # (a profiled step over managed memory can leave the profiler without GPU activity for the rest of the
        # process: the paged optimizer's kernels are those of AdamW8bit, on other addresses)
        if not oname.startswith("Paged"):
            kept.update({f"{oname}/{k}": o for k, o in routes.items()})
    prof = profile_steps(kept)
    for name, (nk, kms) in prof.items():
        oname, k = name.split("/")
        res["optimizers"][oname][k]["kernels_per_step"] = nk
        res["optimizers"][oname][k]["kernel_ms_per_step"] = kms
    for oname, out in res["optimizers"].items():
        line = "  ".join(f"{k} {v['host_ms_median']:.3f} ms ({v.get('kernels_per_step')} kernels, "
                         f"{v.get('kernel_ms_per_step') or 0:.3f} ms)" for k, v in out.items() if isinstance(v, dict))
        print(f"{set_name:9s} {oname:15s} {line}  bitwise={out['grouped_equals_per_parameter_bitwise']}  "
              f"x{out['speedup_host']:.2f}", flush=True)
    del kept
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for optim_step.json")
    ap.add_argument("--sets", default=",".join(SETS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_optim_step.py needs a CUDA device")
    info = device_info()
    print(info, flush=True)
    result = {"info": info, "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "sets": {}}
    for s in args.sets.split(","):
        result["sets"][s] = run_set(s, args)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "optim_step.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
