"""Times Linear8bitLt(4096 -> 11008, threshold=6.0) in eager mode against a CUDA-graph replay of the same layer.

The eager forward materialises the outlier columns with torch.nonzero, a host round trip per call; the captured forward
keeps them on the device.  For M tokens in {1, 16, 256, 4096} and J outlier columns in {0, 5, 41, 100}, each mode is
timed with CUDA events over --calls calls after a warm-up, --repeats times, the two modes alternating (and swapping
which goes first).  Writes int8_graph.json to --out with every sample, the medians, the device name and its power
limit, and whether each replay gave the eager output bit for bit (J <= 64) or within one output ulp plus fp32
accumulation (J > 64).

    python tools/time_int8_graph.py --out <dir>
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitsandbytes_b200 as bnb  # noqa: E402

K, N, THRESHOLD = 4096, 11008, 6.0


def device_info():
    info = {"device": torch.cuda.get_device_name(0), "torch": torch.__version__, "cuda": torch.version.cuda}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def make_layer():
    g = torch.Generator(device="cpu").manual_seed(0)
    lin = torch.nn.Linear(K, N, bias=True)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(N, K, generator=g) * 0.02)
        lin.bias.copy_(torch.randn(N, generator=g) * 0.1)
    layer = bnb.nn.Linear8bitLt(K, N, bias=True, has_fp16_weights=False, threshold=THRESHOLD)
    layer.load_state_dict(lin.state_dict())
    return layer.to("cuda").eval()


def make_input(M, J, seed):
    """fp16 activations below the threshold except J columns, each crossing it in at least one token row."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(M, K, generator=g).clamp_(-5.5, 5.5)
    cols = torch.randperm(K, generator=g)[:J]
    x[torch.randint(M, (J,), generator=g), cols] = 6.5 + 3 * torch.rand(J, generator=g)
    return x.to(torch.float16).cuda()


def time_calls(fn, calls):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e3 / calls  # microseconds per call


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory for int8_graph.json")
    ap.add_argument("--tokens", type=int, nargs="+", default=[1, 16, 256, 4096])
    ap.add_argument("--outliers", type=int, nargs="+", default=[0, 5, 41, 100])
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_int8_graph.py needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    result = {"layer": f"Linear8bitLt({K} -> {N}, threshold={THRESHOLD}, fp16, bias)", "calls": args.calls,
              "repeats": args.repeats, **device_info(), "rows": []}
    layer = make_layer()
    with torch.no_grad():
        for M in args.tokens:
            static_x = make_input(M, 41, seed=M)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                layer(static_x)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_y = layer(static_x)
            for J in args.outliers:
                x = make_input(M, J, seed=1000 * M + J)
                static_x.copy_(x)
                modes = {"eager": lambda: layer(static_x), "graph": graph.replay}
                for fn in modes.values():
                    for _ in range(args.warmup):
                        fn()
                torch.cuda.synchronize()
                eager_out = layer(static_x)
                graph.replay()
                torch.cuda.synchronize()
                if J <= 64:
                    same = bool(torch.equal(eager_out.view(torch.int16), static_y.view(torch.int16)))
                else:  # two fp32 sums in different orders, each rounded to fp16
                    e, g = eager_out.float(), static_y.float()
                    ulp = torch.exp2(torch.floor(torch.log2(torch.maximum(e.abs(), g.abs()).clamp_min(2.0**-14))) - 10)
                    same = bool(((g - e).abs() <= ulp + 2.0**-20 * J**0.5 * (1 + e.abs())).all())
                samples = {name: [] for name in modes}
                for r in range(args.repeats):
                    for name in (("eager", "graph") if r % 2 == 0 else ("graph", "eager")):
                        samples[name].append(time_calls(modes[name], args.calls))
                row = {"M": M, "J": J, "agrees": same,
                       "eager_us": statistics.median(samples["eager"]), "graph_us": statistics.median(samples["graph"]),
                       "eager_samples_us": samples["eager"], "graph_samples_us": samples["graph"]}
                row["speedup"] = row["eager_us"] / row["graph_us"]
                result["rows"].append(row)
                print(f"M={M:5d} J={J:4d}  eager {row['eager_us']:9.1f} us  graph {row['graph_us']:9.1f} us  "
                      f"x{row['speedup']:.2f}  agrees={same}", flush=True)
            del graph, static_y
    with open(os.path.join(args.out, "int8_graph.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(result["device"], "|", result["nvidia_smi"])


if __name__ == "__main__":
    main()
