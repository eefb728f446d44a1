"""Time the grouped LLM.int8() GEMM against the other routes a mixture-of-experts layer on 8-bit experts has.

Shapes (weights quantised row-wise by F.int8_vectorwise_quant, bf16 activations): Mixtral-8x7B gate_up
[8, 28672, 4096] and down [8, 4096, 14336] with top-2 routing, Qwen3-30B-A3B gate_up [128, 1536, 2048] and down
[128, 2048, 768] with top-8 routing; 1, 16, 256 and 4096 tokens, routed by a seeded top-k of uniform router scores;
threshold 0 and 6.0 (activations uniform in [-4, 4] with 8 planted outlier columns per routed token, so that the
outlier preparation runs and is timed).  Routes:

* ``grouped``: bnb.grouped_matmul_8bit, the outlier preparation included;
* ``per_expert_loop``: one Linear8bitLt forward (bnb.matmul with a MatmulLtState) per routed expert, with the splits
  known on the host when the graph is captured;
* ``dequant_all+grouped_mm``: int8_dequant_rows of the whole expert tensor, then torch grouped_mm;
* ``grouped_mm_16bit``: torch grouped_mm on 16-bit experts (no quantisation, the reference point).

Each route's call is captured in a CUDA graph and the replays are timed with CUDA events, so host dispatch stays out of
the numbers.  The card's name, power limit and maximum SM clock are read in the same run and printed first.

    python tools/time_grouped_int8.py --out /tmp/time_grouped_int8
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
THRESHOLDS = (0.0, 6.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--shapes", default=",".join(s[0] for s in SHAPES))
    args = ap.parse_args()

    import torch

    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.autograd._functions import MatmulLtState
    from bitsandbytes_b200.backends.cuda import int8_dequant_rows
    from bitsandbytes_b200.cextension import lib

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")

    def timed(fn):
        """us per replay of fn captured in a CUDA graph."""
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                fn()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fn()
        for _ in range(3):
            graph.replay()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            graph.replay()
        b.record()
        torch.cuda.synchronize()
        lib.check("timed call")
        del graph
        return a.elapsed_time(b) * 1e3 / args.reps

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    rows = []
    wanted = set(args.shapes.split(","))
    torch.set_grad_enabled(False)
    for name, E, N, K, topk in SHAPES:
        if name not in wanted:
            continue
        torch.manual_seed(0)
        W16 = (torch.randn(E, N, K, device=dev) / K**0.5).to(torch.bfloat16)
        CB, SCB, _ = F.int8_vectorwise_quant(W16.to(torch.float16))
        Wt16 = W16.transpose(1, 2)
        for T in TOKENS:
            g = torch.Generator().manual_seed(T)
            choice = torch.rand(T, E, generator=g).topk(topk, dim=1).indices.reshape(-1)
            counts = torch.bincount(choice, minlength=E)
            M = T * topk
            ends = counts.cumsum(0).tolist()
            offs = counts.cumsum(0).to(torch.int32).to(dev)
            x = ((torch.rand(M, K, device=dev, generator=torch.Generator(device=dev).manual_seed(T)) * 2 - 1) * 4)
            x[:, torch.randperm(K, generator=g)[:8].to(dev)] = 7.0
            x = x.to(torch.bfloat16)
            active = int((counts > 0).sum())
            for thr in THRESHOLDS:
                states = []
                for e in range(E):
                    st = MatmulLtState()
                    st.threshold, st.has_fp16_weights, st.is_training = thr, False, False
                    st.CB, st.SCB = CB[e], SCB[e * N:(e + 1) * N]
                    states.append(st)

                def per_expert_loop():
                    s = 0
                    for e, t in enumerate(ends):  # the splits, known on the host at capture
                        if t > s:
                            bnb.matmul(x[s:t], CB[e], state=states[e])
                        s = t

                def dequant_all():
                    Wd = int8_dequant_rows(CB.view(E * N, K), SCB, torch.bfloat16).view(E, N, K)
                    return torch.nn.functional.grouped_mm(x, Wd.transpose(1, 2), offs=offs)

                routes = {"grouped": lambda: bnb.grouped_matmul_8bit(x, CB, SCB, offs, threshold=thr),
                          "per_expert_loop": per_expert_loop,
                          "dequant_all+grouped_mm": dequant_all}
                if thr == 0.0:
                    routes["grouped_mm_16bit"] = lambda: torch.nn.functional.grouped_mm(x, Wt16, offs=offs)
                for route, fn in routes.items():
                    us = timed(fn)
                    r = {"shape": name, "E": E, "N": N, "K": K, "tokens": T, "rows": M, "active_experts": active,
                         "threshold": thr, "route": route, "us": round(us, 2)}
                    rows.append(r)
                    print(json.dumps(r), flush=True)
        del W16, Wt16, CB, SCB
        torch.cuda.empty_cache()
    d = Path(args.out)
    d.mkdir(parents=True, exist_ok=True)
    (d / "time_grouped_int8.json").write_text(json.dumps({"gpu": gpu, "reps": args.reps, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
