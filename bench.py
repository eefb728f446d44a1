#!/usr/bin/env python
"""bench.py -- the headline measurement of BASELINE.json.

    python bench.py --gpus N --steps K --warmup W [--impl reference] [--workload NAME] [--dump-outputs DIR]

A "step" is one pass of the hot path over one batch of synthetic input: the NF4
``Linear4bit`` forward (fused 4-bit dequant GEMM) at a Llama-3-8B linear shape with
bsz x seq = 4096 tokens.  Default workload (BASELINE.json configs[1], the configuration the
metric is quoted on): weight 4096 x 4096, NF4, blocksize 64, bf16, M = 4096.

One JSON line on rank 0:
  value     whole-job TFLOPS with inputs resident in HBM (sum over ranks / max-over-ranks time)
  e2e       same metric through the public module API with HOST (pinned) activations: the
            host->device copy of every step's input and the device->host copy of every step's
            output are inside the timed region (three-stage stream pipeline)
  roofline  dominant kernel vs the measured bf16 tensor peak (MEASURED_PEAKS.json)
  cpu_baseline  the reference CPU path (oracle/_ref, built from the reference sources) on the
            box's host cores, bounded sample, reported beside the GPU number
``--impl reference`` times that CPU reference alone (rank 0 only) and prints the same line shape.

Multi-GPU: the default workload shards by tokens (independent units, no data-path collective):
every rank runs the same layer on its own 4096-token batch -> "scaling": "weak".
The default line also carries
  ref_cuda   the reference's OWN CUDA route for the headline shape on the same box (its dequantize kernel from
             oracle/_ref/libbitsandbytes_cuda_ref.so + cuBLAS, and cuBLAS bf16 alone), measured after the timed region
  secondary  the other BASELINE.json configs (benchmarks/paths.py): configs[1] at M in {1,16,256} and the 11008
             shapes, configs[0] blockwise quantize/dequantize GB/s vs the HBM peak, configs[2] Linear8bitLt,
             configs[4] the Llama-3-8B replica and -- under torchrun -- configs[3] the column-sharded 70B layer.
``--workload blockwise_c1`` / ``int8_c3`` / ``sharded70b`` / ``llama8b`` print those as stand-alone lines;
``--workload optim_f4`` times the optimizer updates of SURVEY.md section 8 row f-4 (not a BASELINE config).
``--no-secondary`` skips them.

``--dump-outputs DIR`` (the c2_* workloads; others reject it) writes, after the timed steps, what the last timed step returned:
DIR/y_rows.npy (float32, 256 seeded rows of the [M, N] output) and DIR/y_row_index.npy (float64, their indices).
The inputs depend only on the arguments (seeded), so two builds can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

WORKLOADS = {
    # name: (N, K, M, quant_type, nested)
    "c2_4096x4096_m4096": (4096, 4096, 4096, "nf4", False),
    "c2_11008x4096_m4096": (11008, 4096, 4096, "nf4", False),
    "c2_4096x11008_m4096": (4096, 11008, 4096, "nf4", False),
    "c2_4096x4096_m256": (4096, 4096, 256, "nf4", False),
    "c2_4096x4096_m16": (4096, 4096, 16, "nf4", False),
    "c2_4096x4096_m1": (4096, 4096, 1, "nf4", False),
}
DEFAULT_WORKLOAD = "c2_4096x4096_m4096"
L2_BYTES = 50 * 1024 * 1024  # H100 SXM


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default=DEFAULT_WORKLOAD)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-secondary", action="store_true")
    ap.add_argument("--layers", type=int, default=32, help="llama8b workload: number of decoder layers")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write a seeded sample of the last timed step's output to DIR/*.npy")
    return ap.parse_args()


# ------------------------------------------------------------------------------------------ clocks
class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons while the timed region runs."""

    FIELDS = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
              "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
              "clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index = index
        self.samples = []
        self._stop = threading.Event()
        self._t = None

    def _loop(self):
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.FIELDS}",
                                      "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=5).stdout
                parts = [p.strip() for p in out.strip().split(",")]
                if len(parts) >= 7:
                    self.samples.append(parts)
            except Exception:
                pass
            self._stop.wait(0.15)

    def __enter__(self):
        self._t = threading.Thread(target=self._loop, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join(timeout=6)
        return False

    def summary(self):
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        sm = sorted(float(s[0]) for s in self.samples if s[0].replace(".", "").isdigit())
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(s[3 + i].lower().startswith("active") for s in self.samples)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": float(self.samples[0][1]),
                "power_w_max": max(float(s[2]) for s in self.samples), "reasons": reasons, "samples": len(self.samples)}


# ------------------------------------------------------------------------------------------ CPU reference arm
def cpu_reference(N, K, M_total, qt, packed_u8, absmax_f32, x_bf16_cpu, budget_s=20.0, steps=1):
    """The reference's CPU implementation of the path (reference backends/cpu/ops.py: native C++
    4-bit dequantize, csrc/cpu_ops.cpp:304-434, then oneDNN F.linear) on all host threads, on a
    bounded row sample of the workload.  Returns (TFLOPS, dict describing the run)."""
    import ctypes as ct

    import torch

    import oracle

    threads = torch.get_num_threads()
    path = oracle.ref_cpu_library_path()
    Wd = torch.empty(N, K, dtype=torch.bfloat16)
    if path is not None:
        kind = "reference"
        lib = ct.CDLL(str(path))
        fn = getattr(lib, f"cdequantize_blockwise_cpu_{qt}_bf16")
        fn.argtypes = [ct.c_void_p, ct.c_void_p, ct.c_void_p, ct.c_longlong, ct.c_longlong, ct.c_longlong]

        def dequant():
            fn(packed_u8.data_ptr(), absmax_f32.data_ptr(), Wd.data_ptr(), 64, N, K)
    else:
        kind = "port"

        def dequant():
            bits = oracle.dequantize_blockwise(packed_u8.numpy(), absmax_f32.numpy(), 64, N * K, qt, None, "bf16")
            Wd.copy_(torch.from_numpy(bits.view("int16")).view(torch.bfloat16).view(N, K))

    def one(m_rows):
        dequant()
        return torch.nn.functional.linear(x_bf16_cpu[:m_rows], Wd)

    # size the sample: start small, grow until one call costs ~budget/ (steps+warm)
    m = min(M_total, 256)
    for _ in range(3):  # page-fault / allocator warm-up (BASELINE.md section 3)
        one(m)
    t0 = time.perf_counter()
    one(m)
    t1 = time.perf_counter() - t0
    target = budget_s / max(steps + 1, 2)
    while m < M_total and t1 * 2.5 < target:
        m = min(M_total, m * 2)
        t0 = time.perf_counter()
        one(m)
        t1 = time.perf_counter() - t0
    times = []
    t_start = time.perf_counter()
    for _ in range(max(steps, 1)):
        t0 = time.perf_counter()
        one(m)
        times.append(time.perf_counter() - t0)
        if time.perf_counter() - t_start > budget_s * 1.5:
            break
    times.sort()
    med = times[len(times) // 2]
    tflops = 2.0 * m * N * K / med / 1e12
    return tflops, {"value": tflops, "unit": "TFLOPS", "cores": threads, "kind": kind,
                    "sample": f"{m} of {M_total} token rows per step (dequantize W + F.linear), median of {len(times)}",
                    "ms_per_sample": med * 1e3}, med, m


def cpu_blockwise_sample(n_total, code_np):
    """cpu_baseline of --workload blockwise_c1: the oracle port (one host thread) dequantising a bounded
    sample of the tensor, blocksize 4096."""
    import numpy as np

    import oracle

    m = 1 << 20
    a = np.random.default_rng(0).standard_normal(m).astype(np.float32)
    codes, absmax = oracle.quantize_blockwise(a, 4096, None, code_np)
    t0 = time.perf_counter()
    reps = 0
    while time.perf_counter() - t0 < 5.0 or reps < 3:
        oracle.dequantize_blockwise(codes, absmax, 4096, m, None, code_np, "fp32")
        reps += 1
    sec = (time.perf_counter() - t0) / reps
    return {"value": (4 * m + m + 4 * m // 4096) / sec / 1e9, "unit": "GB/s", "cores": 1, "kind": "port",
            "sample": f"dequantize_blockwise of {m} of {n_total} elements, blocksize 4096, mean of {reps}"}


def cpu_int8_sample(x_fp16_cpu, cb_np, scb_np, M, N, K):
    """cpu_baseline of --workload int8_c3: the oracle port (one host thread) on 16 token rows: row
    quantisation (threshold 6.0) + int8 GEMM + dequantisation."""
    import numpy as np
    import torch

    import oracle

    rows = 16
    a_bits = x_fp16_cpu[:rows].contiguous().view(torch.int16).numpy().view(np.uint16).reshape(rows, K)
    t0 = time.perf_counter()
    q, stats = oracle.int8_vector_quant(a_bits, 6.0)
    acc = oracle.int8_gemm(q, cb_np)
    oracle.int8_mm_dequant(acc, stats, scb_np)
    sec = time.perf_counter() - t0
    return {"value": 2.0 * rows * N * K / sec / 1e12, "unit": "TOPS", "cores": 1, "kind": "port",
            "sample": f"{rows} of {M} token rows: row quantise + int8 GEMM + dequantise (outlier addmm not included)"}


# ------------------------------------------------------------------------------------------ secondary configs
def secondary_results(dev, args, N, K, M, qt, nested, with_cpu):
    """(ref_cuda, secondary): the reference's CUDA route at the headline shape, and the BASELINE.json configs the
    headline does not cover (rank 0, one GPU, after the timed region).  A failing item reports its error and
    does not take the line down."""
    import torch

    from benchmarks import paths

    ref = paths.load_ref_cuda()
    sec = {}

    def guard(name, fn):
        try:
            sec[name] = fn()
        except Exception as exc:  # noqa: BLE001
            sec[name] = {"error": repr(exc)[:300]}
        torch.cuda.empty_cache()

    ref_cuda = None
    try:
        h = paths.measure_c2(dev, N, K, M, qt, nested, ref=ref, n_calls=40)
        ref_cuda = {"dequant_cublas_us": (h.get("ref_cuda") or {}).get("us"), "cublas_bf16_us": h.get("cublas_bf16_us"),
                    "ours_us": h["us"], "route": (h.get("ref_cuda") or {}).get("route"),
                    "library": "oracle/_ref/libbitsandbytes_cuda_ref.so (built from the reference sources)" if ref else None,
                    "timing": "CUDA-graph replay of 40 back-to-back launches over rotating buffer sets, same process"}
    except Exception as exc:  # noqa: BLE001
        ref_cuda = {"error": repr(exc)[:300]}
    torch.cuda.empty_cache()

    for (n, k, m) in ((4096, 4096, 1), (4096, 4096, 16), (4096, 4096, 256), (11008, 4096, 4096), (4096, 11008, 4096)):
        if (n, k, m) == (N, K, M):
            continue

        def one(n=n, k=k, m=m):
            r = paths.measure_c2(dev, n, k, m, "nf4", False, ref=ref)
            if with_cpu and m < 4096:
                W = (torch.randn(n, k) / k**0.5).to(torch.bfloat16)
                import oracle

                packed, absmax = oracle.quantize_blockwise(W.float().numpy().reshape(-1), 64, "nf4")
                _, info, _, _ = cpu_reference(n, k, m, "nf4", torch.from_numpy(packed), torch.from_numpy(absmax),
                                              torch.randn(m, k).to(torch.bfloat16), budget_s=3.0, steps=3)
                r["cpu_baseline"] = {kk: info[kk] for kk in ("value", "unit", "cores", "kind", "sample")}
            return r

        guard(f"c2_{n}x{k}_m{m}", one)

    def blockwise():
        r = paths.measure_blockwise(dev, ref)
        if with_cpu:
            import bitsandbytes_b200.functional as F

            r["cpu_baseline"] = cpu_blockwise_sample(4 * 1024 * 1024, F.create_dynamic_map().numpy())
        return r

    guard("blockwise_c1", blockwise)

    def int8():
        r = paths.measure_int8_c3(dev)
        cpu_args = r.pop("_cpu_args")
        if with_cpu:
            r["cpu_baseline"] = cpu_int8_sample(*cpu_args)
        return r

    guard("int8_c3", int8)

    def llama():
        from benchmarks.llama import measure_llama8b

        return measure_llama8b(dev, 32, 64)

    guard("llama8b", llama)
    return ref_cuda, sec


# ------------------------------------------------------------------------------------------ output dump
def dump_outputs(out_dir, y, rows=256):
    """The last timed step's output, a fixed seeded sample of its rows, as float32 (and the row indices)."""
    import numpy as np
    import torch

    d = Path(out_dir)
    d.mkdir(parents=True, exist_ok=True)
    idx = np.sort(np.random.default_rng(0).choice(y.shape[0], size=min(rows, y.shape[0]), replace=False))
    sample = y[torch.from_numpy(idx).to(y.device)].float().cpu().numpy()
    np.save(d / "y_rows.npy", sample)
    np.save(d / "y_row_index.npy", idx.astype(np.float64))


# ------------------------------------------------------------------------------------------ main
def _protect_stdout():
    """Native libraries (NCCL's version banner, cuBLAS warnings) write to file descriptor 1; the
    driver wants exactly one JSON line there.  Point fd 1 at stderr and keep Python's sys.stdout
    on the original descriptor."""
    saved = os.dup(1)
    sys.stdout.flush()
    os.dup2(2, 1)
    sys.stdout = os.fdopen(saved, "w", buffering=1)


def main():
    args = parse_args()
    if args.dump_outputs and (args.workload not in WORKLOADS or args.impl != "ours"):
        raise SystemExit(f"--dump-outputs is supported for --impl ours on the {', '.join(WORKLOADS)} workloads only")
    _protect_stdout()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.workload == "sharded70b":
        from benchmarks.sharded import run_sharded70b

        return run_sharded70b(args, rank, world, local_rank)
    if args.workload in ("blockwise_c1", "int8_c3"):
        from benchmarks import paths as bench_paths

        if args.workload == "blockwise_c1":
            return bench_paths.run_blockwise_c1(args, rank, world, local_rank,
                                                None if args.no_cpu_baseline else cpu_blockwise_sample)
        return bench_paths.run_int8_c3(args, rank, world, local_rank, None if args.no_cpu_baseline else cpu_int8_sample)
    if args.workload == "llama8b":
        from benchmarks.llama import run_llama8b

        return run_llama8b(args, rank, world, local_rank)
    if args.workload == "optim_f4":
        from benchmarks.optim import run_optim_f4

        return run_optim_f4(args, rank, world, local_rank)
    N, K, M, qt, nested = WORKLOADS[args.workload]

    import torch

    if args.impl == "reference":
        # the reference's own CPU implementation, rank 0 only, bounded samples
        if rank != 0:
            return
        # torchrun exports OMP_NUM_THREADS=1: the reference arm uses every host core whatever the launcher
        torch.set_num_threads(os.cpu_count() or 1)
        torch.manual_seed(0)
        W = (torch.randn(N, K) / K**0.5).to(torch.bfloat16)
        x = torch.randn(M, K).to(torch.bfloat16)
        import oracle

        packed, absmax = oracle.quantize_blockwise(W.float().numpy().reshape(-1), 64, qt)
        packed_t = torch.from_numpy(packed)
        absmax_t = torch.from_numpy(absmax)
        tflops, info, med, m = cpu_reference(N, K, M, qt, packed_t, absmax_t, x, budget_s=60.0,
                                             steps=max(1, min(args.steps, 20)))
        line = {"impl": "reference", "metric": "nf4_linear4bit_forward_tflops", "value": tflops, "unit": "TFLOPS",
                "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": med * 1e3,
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
                "config": {"workload": args.workload, "N": N, "K": K, "M_per_gpu": M, "global_tokens": M * args.gpus,
                           "quant_type": qt, "blocksize": 64, "double_quant": nested,
                           "parallelism": f"token-sharded replicas x{args.gpus} (no data-path collective)",
                           "l2": "n/a (host run)",
                           "note": "reference CPU backend on host cores; each step is a bounded row sample"},
                "cpu_baseline": {k: info[k] for k in ("value", "unit", "cores", "kind", "sample")},
                "e2e": {"value": tflops, "unit": "TFLOPS", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                "tokens_per_s": m / med}
        print(json.dumps(line), flush=True)
        return

    assert torch.cuda.is_available(), "bench.py needs a CUDA device (the product has no CPU path)"
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist_mod

        dist = dist_mod
        dist.init_process_group("nccl", device_id=dev)

    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.nn import Linear4bit

    torch.manual_seed(0)  # the reference tests' convention; same weights on every rank
    W = (torch.randn(N, K, device=dev) / K**0.5).to(torch.bfloat16)
    layer_bytes = N * K // 2 + 4 * N * K // 64 + 2 * M * K + 2 * M * N
    R = max(2, -(-int(1.25 * L2_BYTES) // layer_bytes))  # rotating sets so that the footprint exceeds L2
    sets = []
    for r in range(R):
        qW, qs = F.quantize_4bit(W, blocksize=64, quant_type=qt, compress_statistics=nested)
        x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        sets.append((qW, qs, x))
    del W
    flops = 2.0 * M * N * K

    def step(i):
        qW, qs, x = sets[i % R]
        return bnb.matmul_4bit(x, qW.t(), qs)

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    for i in range(max(args.warmup, 3)):
        step(i)
    barrier()
    # The K timed steps are captured ONCE into a CUDA graph and replayed inside the timed region (events on the
    # replay's stream, barrier + synchronize on both sides): the K launches run back to back on the device and the
    # per-rank Python / ctypes launch path (5-10 us of jitter per step, which the 8-GPU max-over-ranks time of a
    # 3 ms region otherwise pays) stays outside.  Falls back to an eager loop if capture is not possible.
    graph, side, last = None, torch.cuda.Stream(), None
    try:
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            step(0)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            for i in range(args.steps):
                last = step(i)
        graph.replay()  # one untimed replay: graph upload + allocator warm-up
    except Exception as exc:  # noqa: BLE001
        print(f"[bench] CUDA-graph capture of the timed steps failed ({exc!r}); timing an eager loop", file=sys.stderr)
        graph = None
    barrier()
    e_start, e_end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(local_rank) as clocks:
        t_wall = time.perf_counter()
        e_start.record()
        if graph is not None:
            graph.replay()
        else:
            for i in range(args.steps):
                last = step(i)
        e_end.record()
        barrier()
        t_wall = time.perf_counter() - t_wall
        # At the default K the timed region (~0.3 s) is shorter than a couple of nvidia-smi polls: keep
        # the SAME load running, untimed, until the sampler holds a handful of readings under load.
        t_stop = time.perf_counter() + 2.5
        j = 0
        try:
            while len(clocks.samples) < 6 and time.perf_counter() < t_stop:
                for _ in range(64):
                    step(j)
                    j += 1
                torch.cuda.synchronize()
        except Exception as exc:  # noqa: BLE001  (the continuation only feeds the clock sampler)
            print(f"[bench] clock-sampling continuation stopped: {exc!r}", file=sys.stderr)
        clock_extra_steps = j
    total_ms = e_start.elapsed_time(e_end)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last)
    kernel_ms = total_ms / args.steps  # one kernel per step, launched back to back: the average launch duration
    t = torch.tensor([total_ms], device=dev, dtype=torch.float64)
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    total_ms_max = float(t.item())
    value = world * flops * args.steps / (total_ms_max * 1e-3) / 1e12

    # ---------------------------------------------------------------- e2e through the module API
    layer = Linear4bit(K, N, bias=False, compute_dtype=torch.bfloat16, compress_statistics=nested, quant_type=qt)
    with torch.no_grad():
        layer.weight = bnb.nn.Params4bit((torch.randn(N, K) / K**0.5).to(torch.bfloat16), requires_grad=False,
                                         compress_statistics=nested, quant_type=qt, module=layer)
    layer = layer.to(dev).eval()
    depth = 3
    h_in = [torch.randn(M, K).to(torch.bfloat16).pin_memory() for _ in range(depth)]
    h_out = [torch.empty(M, N, dtype=torch.bfloat16).pin_memory() for _ in range(depth)]
    d_in = [torch.empty(M, K, device=dev, dtype=torch.bfloat16) for _ in range(depth)]
    d_out = [None] * depth
    s_in, s_mm, s_out = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    e_in = [torch.cuda.Event() for _ in range(depth)]
    e_mm = [torch.cuda.Event() for _ in range(depth)]
    e_out = [torch.cuda.Event() for _ in range(depth)]

    def e2e_run(n_steps, timed):
        start = torch.cuda.Event(enable_timing=True)
        end = torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record(s_in)
        for i in range(n_steps):
            b = i % depth
            with torch.cuda.stream(s_in):
                if i >= depth:
                    s_in.wait_event(e_mm[b])       # the GEMM that read d_in[b] is done
                d_in[b].copy_(h_in[b], non_blocking=True)
                e_in[b].record(s_in)
            with torch.cuda.stream(s_mm), torch.no_grad():
                s_mm.wait_event(e_in[b])
                if i >= depth:
                    s_mm.wait_event(e_out[b])      # the D2H that read d_out[b] is done
                d_out[b] = layer(d_in[b])
                e_mm[b].record(s_mm)
            with torch.cuda.stream(s_out):
                s_out.wait_event(e_mm[b])
                h_out[b].copy_(d_out[b], non_blocking=True)
                e_out[b].record(s_out)
        s_out.wait_stream(s_mm)
        s_out.wait_stream(s_in)
        end.record(s_out)
        torch.cuda.synchronize()
        return start.elapsed_time(end)

    e2e_run(max(args.warmup, 3), False)
    barrier()
    e2e_ms = e2e_run(args.steps, True)
    t = torch.tensor([e2e_ms], device=dev, dtype=torch.float64)
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e_value = world * flops * args.steps / (float(t.item()) * 1e-3) / 1e12

    # ---------------------------------------------------------------- configs[3] under torchrun (all ranks)
    sharded = None
    if dist is not None and not args.no_secondary:
        try:
            from benchmarks.sharded import measure_sharded70b

            sets = None
            torch.cuda.empty_cache()
            sharded = measure_sharded70b(dev, rank, world, max(10, min(args.steps, 50)), args.warmup)
        except Exception as exc:  # noqa: BLE001
            sharded = {"error": repr(exc)[:300]}

    if rank != 0:
        if dist is not None:
            dist.destroy_process_group()
        return

    # ---------------------------------------------------------------- roofline + CPU baseline
    peaks = {}
    try:
        peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
    except Exception:
        pass
    long_loop = total_ms_max > 2000.0
    if peaks:
        peak = peaks["bf16_tflops_sustained"] if long_loop else peaks["bf16_tflops"]
        peak_src = "MEASURED_PEAKS.json " + ("bf16_tflops_sustained" if long_loop else "bf16_tflops (burst)")
    else:
        peak, peak_src = 989.0, "H100 SXM data sheet, dense bf16 (not a measured peak)"
    achieved = flops / (kernel_ms * 1e-3) / 1e12
    traffic, traffic_src, kernel_name = None, None, "gemm4_tc_kernel<bf16, NF4> (wgmma)"
    roofline = {"bound": "tensor", "achieved": achieved, "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak,
                "traffic": traffic, "traffic_source": traffic_src, "peak_source": peak_src, "kernel": kernel_name,
                "kernel_ms": kernel_ms}

    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        qW, qs, x = sets[0]
        _, cpu, _, _ = cpu_reference(N, K, M, qt, qW.reshape(-1).cpu(), qs.absmax.cpu(), x.cpu(), budget_s=15.0, steps=5)
        cpu = {k: cpu[k] for k in ("value", "unit", "cores", "kind", "sample")}
    sets = None
    torch.cuda.empty_cache()

    # ---------------------------------------------------------------- the reference's CUDA route + the other configs
    ref_cuda, secondary = None, None
    if not args.no_secondary:
        ref_cuda, secondary = secondary_results(dev, args, N, K, M, qt, nested, world == 1 and not args.no_cpu_baseline)
        if sharded is not None:
            secondary["sharded70b"] = sharded

    line = {
        "metric": "nf4_linear4bit_forward_tflops", "value": value, "unit": "TFLOPS", "n_gpus": world,
        "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": total_ms_max / args.steps,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": {"workload": args.workload, "N": N, "K": K, "M_per_gpu": M, "global_tokens": M * world,
                   "quant_type": qt, "blocksize": 64, "double_quant": nested,
                   "parallelism": f"token-sharded replicas x{world} (no data-path collective)",
                   "l2": f"rotating {R} buffer sets ({R * layer_bytes / 2**20:.0f} MiB > {L2_BYTES >> 20} MiB L2)"},
        "tokens_per_s": world * M * args.steps / (total_ms_max * 1e-3),
        "e2e": {"value": e2e_value, "unit": "TFLOPS", "h2d_bytes_per_step": 2 * M * K, "d2h_bytes_per_step": 2 * M * N,
                "api": "bitsandbytes_b200.nn.Linear4bit.forward on pinned-host activations, 3-stage stream pipeline"},
        "gpu_launches": args.steps,
        "timed_region": "CUDA-graph replay of the K steps" if graph is not None else "eager loop of the K steps",
        "roofline": roofline,
        "cpu_baseline": cpu,
        "ref_cuda": ref_cuda,
        "secondary": secondary,
        "clocks": dict(clocks.summary(), window=f"timed region + {clock_extra_steps} untimed steps of the same loop"),
        "wall_s": t_wall,
    }
    print(json.dumps(line), flush=True)
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
