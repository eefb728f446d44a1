"""Shared helpers of the bench workloads (top-level bench code: not part of the product package)."""
from __future__ import annotations

import json
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
L2_BYTES = 50 * 1024 * 1024  # H100 SXM


def peaks():
    try:
        return json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
    except Exception:  # noqa: BLE001
        return {}


def hbm_peak():
    p = peaks()
    if "hbm_gbs" in p:
        return float(p["hbm_gbs"]), "MEASURED_PEAKS.json hbm_gbs"
    return 3350.0, "H100 SXM data sheet HBM3 bandwidth (not a measured peak)"


def bf16_peak(sustained=False):
    p = peaks()
    key = "bf16_tflops_sustained" if sustained else "bf16_tflops"
    if key in p:
        return float(p[key]), f"MEASURED_PEAKS.json {key}" + ("" if sustained else " (burst)")
    return 989.0, "H100 SXM data sheet, dense bf16 (not a measured peak)"


def sets_for(bytes_per_set: int, minimum: int = 2) -> int:
    """Number of rotating buffer sets so that the footprint exceeds L2 (no flush needed between launches)."""
    return max(minimum, -(-int(1.25 * L2_BYTES) // max(1, bytes_per_set)))


def time_us(fn, n_calls: int, warmup: int = 3, use_graph: bool = True, rounds: int = 5):
    """Microseconds per call of fn(i), device-timed with CUDA events.

    The calls are captured ONCE into a CUDA graph (n_calls back-to-back launches over the caller's rotating
    buffer sets) and the graph is replayed `rounds` times; the median replay is reported.  This removes the
    host launch path (ctypes + Python, 5-10 us per call) from the measurement of 5-50 us kernels.  Ops that
    cannot be captured (host synchronisation inside) fall back to an eager back-to-back loop.
    Returns (us_per_call, mode)."""
    import torch

    for i in range(max(warmup, 3)):
        fn(i)
    torch.cuda.synchronize()
    if use_graph:
        try:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                fn(0)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                for i in range(n_calls):
                    fn(i)
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            ts = []
            for _ in range(rounds):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3 / n_calls)
            ts.sort()
            return ts[len(ts) // 2], "cuda-graph"
        except Exception:  # noqa: BLE001
            torch.cuda.synchronize()
    ts = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n_calls):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / n_calls)
    ts.sort()
    return ts[len(ts) // 2], "eager"
