"""Measurements of the BASELINE.json configs beside the headline one, each returning a small dict that bench.py
prints as its own line (``--workload NAME``) and also folds into the default line's ``secondary`` object:

  c2        configs[1] at every token count / shape: ``bnb.matmul_4bit`` NF4 at M in {1,16,256,4096}
  blockwise configs[0] on the GPU: quantize_blockwise / dequantize_blockwise, 4 Mi fp32 elements (blocksize 4096,
            256), a 256 Mi-element tensor for the asymptote, and the NF4 weight (4096 x 4096 bf16, blocksize 64)
  int8_c3   configs[2]: ``Linear8bitLt`` (LLM.int8(), threshold 6.0) forward, 4096 -> 11008, 4096 tokens, fp16,
            five outlier columns (reference benchmarking/matmul_benchmark.py:47-48)

Every figure is device-timed (CUDA events around a CUDA-graph replay of back-to-back launches over rotating
buffer sets larger than L2; see common.time_us).  ``ref_cuda`` numbers are the REFERENCE's own CUDA library,
built from its sources into oracle/_ref (same C ABI), driven on the same buffers in the same process along
the route the reference takes on this GPU (reference_uses_fused: its sm_90 rule, fused kernel or dequantize +
cuBLAS).  This is top-level bench code; the product package never imports oracle/.
"""
from __future__ import annotations

import ctypes as ct

from .common import L2_BYTES, bf16_peak, hbm_peak, sets_for, time_us

_QT = {"fp4": 1, "nf4": 2}


def load_ref_cuda():
    """The reference CUDA library (oracle/_ref/libbitsandbytes_cuda_ref.so) or None."""
    try:
        import oracle

        path = oracle.ref_cuda_library_path()
        if path is None or not path.exists():
            return None
        return ct.CDLL(str(path))
    except Exception:  # noqa: BLE001
        return None


def _stream():
    import torch

    return ct.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else ct.c_void_p(t.data_ptr())


def reference_uses_fused(M, N, K):
    """Whether the reference takes its fused kernel (True) or dequantise + cuBLAS (False) for a 16-bit GEMM on this
    device: its backends/cuda/ops.py:_gemm_4bit_use_custom_cuda for sm_90 (the H100 branch, ops.py:600-603,
    629-680, 745-755), with the SM count read from the device, and its M <= 1536 cap (ops.py:926)."""
    import torch

    if M <= 4:
        return True
    if M > 1536:
        return False
    num_sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    n_blocks = (N + 63) // 64
    if N * K < 4 * 1024 * 1024:  # small weights
        if K * 2 < N:
            return M <= (512 if n_blocks * 3 < num_sms else 320)
        if n_blocks * 4 <= num_sms:
            return M <= 32
        if n_blocks * 2 <= num_sms:
            return M <= 16
        return False
    if M > 512:
        return False
    if M < 8:
        if M >= 6 and n_blocks >= 36:
            lt_75 = n_blocks * 4 < num_sms * 3
            lt_60 = n_blocks * 5 < num_sms * 3
            if K > N and lt_75:
                return False
            if K == N and lt_75 and not lt_60:
                return False
        return True
    if n_blocks >= num_sms * 3:
        return M <= 64
    if n_blocks >= num_sms * 2:
        return M <= 48
    if n_blocks >= num_sms:
        return M <= 32
    if n_blocks >= num_sms // 2:
        if K >= N and n_blocks * 4 < num_sms * 3:
            return False
        return M <= 16
    return False


# ------------------------------------------------------------------------------------------ configs[1]
def measure_c2(dev, N, K, M, qt="nf4", nested=False, ref=None, n_calls=None, with_cublas=True):
    import torch

    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    torch.manual_seed(0)
    W = (torch.randn(N, K, device=dev) / K**0.5).to(torch.bfloat16)
    layer_bytes = N * K // 2 + 4 * N * K // 64 + 2 * M * K + 2 * M * N
    R = sets_for(layer_bytes)
    sets = []
    for _ in range(R):
        qW, qs = F.quantize_4bit(W, blocksize=64, quant_type=qt, compress_statistics=nested)
        x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        sets.append((qW, qs, x, out))
    flops = 2.0 * M * N * K
    if n_calls is None:
        n_calls = max(R, min(200, int(4e9 // max(flops / 1e3, 1)) or 1))
        n_calls = max(R, min(n_calls, 100))

    def ours(i):
        qW, qs, x, out = sets[i % R]
        bnb.matmul_4bit(x, qW.t(), qs)

    us, mode = time_us(ours, n_calls)
    res = {"N": N, "K": K, "M": M, "quant_type": qt, "double_quant": nested, "us": us, "tflops": flops / us / 1e6,
           "tokens_per_s": M / (us * 1e-6), "timing": mode, "sets": R}
    algo_bytes = layer_bytes
    tpeak, tsrc = bf16_peak()
    hpeak, hsrc = hbm_peak()
    t_tensor = flops / (tpeak * 1e6)       # us at the tensor peak
    t_hbm = algo_bytes / (hpeak * 1e3)     # us at the HBM peak
    if t_tensor >= t_hbm:
        res["roofline"] = {"bound": "tensor", "achieved": flops / us / 1e6, "peak": tpeak, "unit": "TFLOP/s",
                           "frac": flops / us / 1e6 / tpeak, "peak_source": tsrc}
    else:
        res["roofline"] = {"bound": "hbm", "achieved": algo_bytes / us / 1e3, "peak": hpeak, "unit": "GB/s",
                           "frac": algo_bytes / us / 1e3 / hpeak, "peak_source": hsrc, "algorithmic_bytes": algo_bytes}

    if with_cublas:
        Wd = torch.empty(N, K, device=dev, dtype=torch.bfloat16)

        def cublas(i):
            _, _, x, out = sets[i % R]
            torch.matmul(x, Wd.t(), out=out)

        cu_us, _ = time_us(cublas, n_calls)
        res["cublas_bf16_us"] = cu_us
    if ref is not None and not nested:
        Wd = torch.empty(N, K, device=dev, dtype=torch.bfloat16)
        fused = reference_uses_fused(M, N, K)
        deq = getattr(ref, f"cdequantize_blockwise_bf16_{qt}")
        gemm = getattr(ref, "cgemm_4bit_bf16", None)

        def ref_route(i):
            qW, qs, x, out = sets[i % R]
            if fused and gemm is not None:
                gemm(_p(x), _p(qW), _p(qs.absmax), None, None, None, _p(out), None, M, N, K, 64, _QT[qt], _stream())
            else:
                deq(None, _p(qW), _p(qs.absmax), _p(Wd), 64, N * K, _stream())
                torch.matmul(x, Wd.t(), out=out)

        r_us, r_mode = time_us(ref_route, n_calls)
        res["ref_cuda"] = {"us": r_us, "route": "fused cgemm_4bit_bf16" if fused and gemm is not None else
                           "cdequantize_blockwise_bf16 + cuBLAS (F.linear)", "tflops": flops / r_us / 1e6,
                           "timing": r_mode, "speedup_ours": r_us / us}
    return res


# ------------------------------------------------------------------------------------------ configs[0]
def measure_blockwise(dev, ref=None, asymptote=True):
    import torch

    import bitsandbytes_b200.functional as F

    peak, peak_src = hbm_peak()
    code = F.create_dynamic_map().to(dev)
    results = {}

    def bw8(n, bs, tag):
        per_set = n * 9
        R = sets_for(per_set, 2) if n <= (1 << 26) else 2
        As = [torch.randn(n, device=dev) for _ in range(R)]
        qs = [F.quantize_blockwise(a, code=code, blocksize=bs) for a in As]
        outs = [torch.empty(n, device=dev) for _ in range(R)]
        q_out = [torch.empty(n, device=dev, dtype=torch.uint8) for _ in range(R)]
        q_abs = [torch.empty(-(n // -bs), device=dev) for _ in range(R)]
        algo = 4 * n + n + 4 * (n // bs)
        n_calls = max(R, min(60, int(3e9 // algo) + 1))

        def quant(i):
            F.quantize_blockwise(As[i % R], code=code, blocksize=bs)

        def dequant(i):
            q, st = qs[i % R]
            F.dequantize_blockwise(q, st, out=outs[i % R])

        for name, fn in (("quantize", quant), ("dequantize", dequant)):
            us, mode = time_us(fn, n_calls)
            results[f"{name}_{tag}"] = {"elements": n, "blocksize": bs, "us": us, "gb_per_s": algo / us / 1e3,
                                        "frac_of_hbm_peak": algo / us / 1e3 / peak, "algorithmic_bytes": algo,
                                        "timing": mode}
        if ref is not None:
            def rquant(i):
                ref.cquantize_blockwise_fp32(_p(code), _p(As[i % R]), _p(q_abs[i % R]), _p(q_out[i % R]), bs, n)

            def rdequant(i):
                q, st = qs[i % R]
                ref.cdequantize_blockwise_fp32(_p(code), _p(q), _p(st.absmax), _p(outs[i % R]), bs, n, _stream())

            us, _ = time_us(rquant, n_calls, use_graph=False)  # the reference quantize has no stream argument
            results[f"quantize_{tag}"]["ref_cuda_us"] = us
            us, _ = time_us(rdequant, n_calls)
            results[f"dequantize_{tag}"]["ref_cuda_us"] = us
        del As, qs, outs, q_out, q_abs
        torch.cuda.empty_cache()

    n = 4 * 1024 * 1024
    bw8(n, 4096, "fp32_4Mi_bs4096")
    bw8(n, 256, "fp32_4Mi_bs256")
    if asymptote:
        bw8(256 * 1024 * 1024, 4096, "fp32_256Mi_bs4096")

    # NF4 weight of configs[1]: 4096 x 4096 bf16, blocksize 64 (what Linear4bit quantises / dequantises)
    N = K = 4096
    nw = N * K
    per_set = nw * 2 + nw // 2 + 4 * nw // 64
    R = sets_for(per_set)
    Ws = [torch.randn(N, K, device=dev, dtype=torch.bfloat16) for _ in range(R)]
    qs = [F.quantize_4bit(w, blocksize=64, quant_type="nf4") for w in Ws]
    outs = [torch.empty(N, K, device=dev, dtype=torch.bfloat16) for _ in range(R)]
    q_out = [torch.empty((nw // 2, 1), device=dev, dtype=torch.uint8) for _ in range(R)]
    q_abs = [torch.empty(nw // 64, device=dev) for _ in range(R)]
    algo = per_set

    def q4(i):
        F.quantize_4bit(Ws[i % R], blocksize=64, quant_type="nf4")

    def d4(i):
        q, st = qs[i % R]
        F.dequantize_4bit(q, st, out=outs[i % R])

    for name, fn in (("quantize", q4), ("dequantize", d4)):
        us, mode = time_us(fn, 40)
        results[f"{name}_nf4_bf16_4096x4096_bs64"] = {"elements": nw, "blocksize": 64, "us": us, "gb_per_s": algo / us / 1e3,
                                                     "frac_of_hbm_peak": algo / us / 1e3 / peak, "algorithmic_bytes": algo,
                                                     "timing": mode}
    if ref is not None:
        def rq4(i):
            ref.cquantize_blockwise_bf16_nf4(None, _p(Ws[i % R]), _p(q_abs[i % R]), _p(q_out[i % R]), 64, nw)

        def rd4(i):
            q, st = qs[i % R]
            ref.cdequantize_blockwise_bf16_nf4(None, _p(q), _p(st.absmax), _p(outs[i % R]), 64, nw, _stream())

        us, _ = time_us(rq4, 40, use_graph=False)
        results["quantize_nf4_bf16_4096x4096_bs64"]["ref_cuda_us"] = us
        us, _ = time_us(rd4, 40)
        results["dequantize_nf4_bf16_4096x4096_bs64"]["ref_cuda_us"] = us
    return {"peak_gb_per_s": peak, "peak_source": peak_src, "results": results}


# ------------------------------------------------------------------------------------------ configs[2]
def measure_int8_c3(dev, steps=40):
    import torch

    import bitsandbytes_b200 as bnb

    K, N, M = 4096, 11008, 4096
    torch.manual_seed(0)
    lin = torch.nn.Linear(K, N, bias=False)
    layer = bnb.nn.Linear8bitLt(K, N, bias=False, has_fp16_weights=False, threshold=6.0)
    layer.load_state_dict(lin.state_dict())
    layer = layer.to(dev).eval()  # quantises the weight to int8 + SCB on the move to the device
    outlier_cols = torch.randint(0, K, (5,), generator=torch.Generator().manual_seed(1)).tolist()
    sets = 3  # activations 32 MiB + outputs 86 MiB per set: 3 sets exceed the 50 MiB L2
    xs = []
    for _ in range(sets):
        x = torch.randn(M, K, device=dev, dtype=torch.float16)
        x[:, outlier_cols] = 8.0
        xs.append(x)
    with torch.no_grad():
        def fwd(i):
            return layer(xs[i % sets])

        us, mode = time_us(fwd, max(6, min(steps, 60)), use_graph=False)  # the outlier-column lookup syncs with the host
        xs0 = [torch.randn(M, K, device=dev, dtype=torch.float16).clamp_(-5.5, 5.5) for _ in range(sets)]

        def fwd0(i):
            return layer(xs0[i % sets])

        us0, _ = time_us(fwd0, max(6, min(steps, 60)), use_graph=False)
        # the fp16 layer the reference benchmark compares with (cuBLAS)
        w16 = lin.weight.detach().to(dev, torch.float16)

        def fp16(i):
            return torch.nn.functional.linear(xs[i % sets], w16)

        us16, _ = time_us(fp16, 20)
    ops = 2.0 * M * N * K
    CB = layer.state.CB if layer.state.CB is not None else layer.weight.CB
    SCB = layer.state.SCB if layer.state.SCB is not None else layer.weight.SCB
    return {"N": N, "K": K, "M": M, "threshold": 6.0, "outlier_columns": len(set(outlier_cols)), "us": us,
            "tops": ops / us / 1e6, "tokens_per_s": M / (us * 1e-6), "us_no_outliers": us0, "fp16_cublas_linear_us": us16,
            "timing": mode, "api": "bitsandbytes_b200.nn.Linear8bitLt.forward",
            "_cpu_args": (xs[0].cpu(), CB.cpu().numpy(), SCB.float().cpu().numpy(), M, N, K)}


# ------------------------------------------------------------------------------------------ stand-alone lines
def run_blockwise_c1(args, rank, world, local_rank, cpu_baseline=None):
    import json

    import torch

    if rank != 0:
        return
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    r = measure_blockwise(dev, load_ref_cuda())
    head = r["results"]["dequantize_fp32_4Mi_bs4096"]
    import bitsandbytes_b200.functional as F

    cpu = cpu_baseline(4 * 1024 * 1024, F.create_dynamic_map().numpy()) if cpu_baseline is not None else None
    line = {"metric": "blockwise_dequantize_fp32_gb_per_s", "value": head["gb_per_s"], "unit": "GB/s", "n_gpus": 1,
            "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": head["us"] * 1e-3, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic (randn, seed 0)",
            "config": {"workload": "blockwise_c1", "elements": 4 * 1024 * 1024, "blocksizes": [4096, 256],
                       "l2": "rotating buffer sets larger than the 50 MiB L2"},
            "results": r["results"],
            "roofline": {"bound": "hbm", "achieved": head["gb_per_s"], "peak": r["peak_gb_per_s"], "unit": "GB/s",
                         "frac": head["gb_per_s"] / r["peak_gb_per_s"], "traffic": None, "peak_source": r["peak_source"],
                         "kernel": "dequantize_blockwise_kernel<float, 8-bit>"},
            "cpu_baseline": cpu, "gpu_launches": None, "e2e": None}
    print(json.dumps(line), flush=True)


def run_int8_c3(args, rank, world, local_rank, cpu_baseline=None):
    import json

    import torch

    if rank != 0:
        return
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    r = measure_int8_c3(dev, args.steps)
    cpu_args = r.pop("_cpu_args")
    cpu = cpu_baseline(*cpu_args) if cpu_baseline is not None else None
    line = {"metric": "linear8bitlt_forward_tops", "value": r["tops"], "unit": "TOPS", "n_gpus": 1, "steps": args.steps,
            "warmup": max(args.warmup, 3), "ms_per_step": r["us"] * 1e-3, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "int8 (fp16 activations, fp16 outlier columns)",
            "data": "synthetic (randn, seed 0)", "config": dict(workload="int8_c3", **{k: r[k] for k in
                                                                    ("N", "K", "M", "threshold", "outlier_columns", "api")}),
            "results": r, "tokens_per_s": r["tokens_per_s"], "cpu_baseline": cpu, "gpu_launches": None, "e2e": None}
    print(json.dumps(line), flush=True)
