#!/usr/bin/env python
"""Generate the golden fixtures in tests/golden/ by running the REFERENCE itself.

Run here (the build container), never on the GPU box: it imports the reference Python
package from /root/reference (read-only).  The reference looks for its native library
inside its own package directory, so the script assembles a throw-away package under a
temp dir made of symlinks to the reference's files -- nothing of the reference is copied
into this repository; only the small .npz written next to this script is committed.

Two phases, each in its own interpreter (the reference registers its kernels at import):

  native   the package sees oracle/_ref/libbitsandbytes_cpu.so (built from the reference
           sources by oracle/Makefile): outputs of the reference's C++ CPU backend
           (csrc/cpu_ops.cpp) -- dequantize (8-bit / NF4 / FP4), LUT-approximate 8-bit
           quantize, and bnb.matmul_4bit / F.dequantize_4bit through the public API.
  default  no native library: the dispatcher falls through to the reference's pure-PyTorch
           "default" kernels (bitsandbytes/backends/default/ops.py), which are the executable
           statement of the CUDA semantics for quantize (exact nearest code, ties to the
           lower index) and for the LLM.int8() ops.

    python tests/golden/make_golden.py

Everything is seeded with torch.manual_seed(0), the reference tests' own convention
(reference tests/conftest.py:9-14).
"""
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
REPO = HERE.parent.parent
REF = Path(os.environ.get("BNB_REFERENCE_DIR", "/root/reference"))
DT_NAME = {torch.bfloat16: "bf16", torch.float16: "fp16", torch.float32: "fp32"}


def import_reference(with_native: bool):
    tmp = Path(tempfile.mkdtemp(prefix="bnbref_"))
    pkg = tmp / "bitsandbytes"

    def mirror(src: Path, dst: Path):
        dst.mkdir()
        for p in src.iterdir():
            if p.name == "__pycache__":
                continue
            if p.is_dir():
                mirror(p, dst / p.name)
            else:
                (dst / p.name).symlink_to(p)

    mirror(REF / "bitsandbytes", pkg)
    if with_native:
        lib = REPO / "oracle" / "_ref" / "libbitsandbytes_cpu.so"
        if not lib.exists():
            raise SystemExit("build oracle/_ref first: make -C oracle ref-cpu")
        (pkg / "libbitsandbytes_cpu.so").symlink_to(lib)
    sys.path.insert(0, str(tmp))
    sys.dont_write_bytecode = True
    import bitsandbytes as bnb

    assert Path(bnb.__file__).parent == pkg
    return bnb


def bits(t: torch.Tensor) -> np.ndarray:
    """16-bit float tensors travel as uint16 bit patterns; everything else as-is."""
    t = t.detach().contiguous()
    if t.dtype in (torch.bfloat16, torch.float16):
        return t.view(torch.int16).numpy().view(np.uint16).copy()
    return t.numpy().copy()


def make_inputs():
    """Seeded inputs shared by both phases (same order of RNG draws)."""
    torch.manual_seed(0)
    inp = {}
    for name, n, bs in (("a", 8192, 256), ("b", 4096 * 2 + 37, 4096), ("c", 1000, 64)):
        A = torch.randn(n, dtype=torch.float32)
        A[5] = 0.0
        inp[f"q8_{name}"] = (A, bs)
    for name, shape, bs, dt in (
        ("a", (64, 128), 64, torch.bfloat16),
        ("b", (4097,), 32, torch.float32),
        ("c", (48, 256), 128, torch.float16),
    ):
        inp[f"q4_{name}"] = (torch.randn(*shape, dtype=torch.float32).to(dt), bs, shape, dt)
    for name, (M, N, K), qt, nested, dt, with_bias in (
        ("plain", (5, 48, 128), "nf4", False, torch.bfloat16, False),
        ("nested", (3, 512, 128), "fp4", True, torch.bfloat16, True),
        ("fp16", (2, 40, 192), "nf4", False, torch.float16, True),
    ):
        W = (torch.randn(N, K) / K**0.5).to(dt)
        x = torch.randn(M, K).to(dt)
        bias = torch.randn(N).to(dt) if with_bias else None
        inp[f"gemm4_{name}"] = (W, x, bias, qt, nested, dt, (M, N, K))
    A = torch.randn(7, 96).half()
    A[:, 11] = 8.5
    A[2, 40] = -7.0
    inp["i8vq"] = A
    inp["i8mm"] = (
        torch.randint(-127, 128, (9, 64), dtype=torch.int8),
        torch.randint(-127, 128, (24, 64), dtype=torch.int8),
        torch.rand(9) * 3 + 0.1,
        torch.rand(24) * 2 + 0.1,
        torch.randn(24).half(),
    )
    # later additions draw AFTER everything above, so the earlier cases keep their values
    for name, n, bs in (("d", 1, 256), ("e", 255, 256), ("f", 4096 * 3, 512), ("g", 70001, 2048), ("h", 129, 64)):
        inp[f"q8_{name}"] = (torch.randn(n, dtype=torch.float32) * (10.0 if name == "g" else 1.0), bs)
    for name, shape, bs, dt in (
        ("d", (1,), 64, torch.float32),
        ("e", (63,), 64, torch.bfloat16),
        ("f", (3, 1000), 256, torch.float16),
        ("g", (16, 4096), 4096, torch.bfloat16),
        ("h", (130,), 32, torch.float32),
        ("i", (5, 512), 512, torch.float32),
    ):
        inp[f"q4_{name}"] = (torch.randn(*shape, dtype=torch.float32).to(dt), bs, shape, dt)
    return inp


Q8_NAMES = ("a", "b", "c", "d", "e", "f", "g", "h")
Q4_NAMES = ("a", "b", "c", "d", "e", "f", "g", "h", "i")


def phase(which: str, out_path: str):
    bnb = import_reference(with_native=(which == "native"))
    F = bnb.functional
    ops = torch.ops.bitsandbytes
    inp = make_inputs()
    out = {}
    code = F.create_dynamic_map()

    if which == "default":
        out["dynamic_map"] = code.numpy()
        out["nf4_code"] = F.get_4bit_type("nf4", device="cpu").numpy()
        out["fp4_code"] = F.get_4bit_type("fp4", device="cpu").numpy()

    for name in Q8_NAMES:
        A, bs = inp[f"q8_{name}"]
        q, absmax = ops.quantize_blockwise(A, code, bs)
        key = f"q8_{name}"
        if which == "default":
            out[f"{key}_A"] = A.numpy()
            out[f"{key}_bs"] = np.int64(bs)
            out[f"{key}_codes"] = q.numpy()
            out[f"{key}_absmax"] = absmax.numpy()
        else:
            out[f"{key}_codes_cpulib"] = q.numpy()
            out[f"{key}_absmax_cpulib"] = absmax.numpy()
        # each phase dequantizes its own codes (default: torch kernel; native: C++ kernel)
        for dt in (torch.float32, torch.bfloat16, torch.float16):
            d = ops.dequantize_blockwise(q, absmax, code, bs, dt)
            out[f"{key}_deq_{DT_NAME[dt]}_{which}"] = bits(d)

    for qt in ("nf4", "fp4"):
        for name in Q4_NAMES:
            A, bs, shape, dt = inp[f"q4_{name}"]
            key = f"q4_{qt}_{name}"
            packed, absmax = ops.quantize_4bit(A, bs, qt, torch.uint8)  # default impl in both phases
            if which == "default":
                out[f"{key}_A"] = bits(A)
                out[f"{key}_dtype"] = np.array(DT_NAME[dt])
                out[f"{key}_bs"] = np.int64(bs)
                out[f"{key}_packed"] = packed.reshape(-1).numpy()
                out[f"{key}_absmax"] = absmax.numpy()
            for odt in (torch.float32, torch.bfloat16, torch.float16):
                d = ops.dequantize_4bit(packed, absmax, bs, qt, list(shape), odt)
                out[f"{key}_deq_{DT_NAME[odt]}_{which}"] = bits(d.reshape(-1))

    if which == "native":
        for name in ("plain", "nested", "fp16"):
            W, x, bias, qt, nested, dt, (M, N, K) = inp[f"gemm4_{name}"]
            qW, qs = F.quantize_4bit(W, blocksize=64, quant_type=qt, compress_statistics=nested)
            y = bnb.matmul_4bit(x, qW.t(), qs, bias=bias)
            Wdq = F.dequantize_4bit(qW, qs)
            key = f"gemm4_{name}"
            out[f"{key}_x"] = bits(x)
            out[f"{key}_packed"] = qW.reshape(-1).numpy()
            out[f"{key}_shape"] = np.array([M, N, K], np.int64)
            out[f"{key}_qt"] = np.array(qt)
            out[f"{key}_dtype"] = np.array(DT_NAME[dt])
            if nested:
                out[f"{key}_absmax8"] = qs.absmax.numpy()
                out[f"{key}_absmax2"] = qs.state2.absmax.numpy()
                out[f"{key}_code2"] = qs.state2.code.numpy()
                out[f"{key}_offset"] = qs.offset.numpy().reshape(1)
            else:
                out[f"{key}_absmax"] = qs.absmax.numpy()
            if bias is not None:
                out[f"{key}_bias"] = bits(bias)
            out[f"{key}_Wdq"] = bits(Wdq.reshape(-1))
            out[f"{key}_y"] = bits(y.reshape(-1))
    else:
        A = inp["i8vq"]
        for thr, tag in ((0.0, "t0"), (6.0, "t6")):
            qa, stats, oc = ops.int8_vectorwise_quant(A, thr)
            out[f"i8vq_{tag}_A"] = bits(A)
            out[f"i8vq_{tag}_q"] = qa.numpy()
            out[f"i8vq_{tag}_stats"] = stats.numpy()
            out[f"i8vq_{tag}_cols"] = (oc if oc is not None else torch.empty(0, dtype=torch.int64)).numpy()
        Ai, Bi, rs, cs, bias = inp["i8mm"]
        Ci = ops.int8_linear_matmul(Ai, Bi)
        out["i8mm_A"] = Ai.numpy()
        out["i8mm_B"] = Bi.numpy()
        out["i8mm_C"] = Ci.numpy()
        out["i8mm_rs"] = rs.numpy()
        out["i8mm_cs"] = cs.numpy()
        out["i8mm_bias"] = bits(bias)
        out["i8mm_deq_nobias"] = bits(ops.int8_mm_dequant(Ci, rs, cs, dtype=torch.float16))
        out["i8mm_deq_bias"] = bits(ops.int8_mm_dequant(Ci, rs, cs, dtype=torch.float16, bias=bias))

    out[f"reference_version_{which}"] = np.array(bnb.__version__)
    np.savez(out_path, **out)


def main():
    if len(sys.argv) == 4 and sys.argv[1] == "--phase":
        phase(sys.argv[2], sys.argv[3])
        return
    merged = {}
    with tempfile.TemporaryDirectory() as td:
        for which in ("default", "native"):
            p = os.path.join(td, f"{which}.npz")
            subprocess.run([sys.executable, __file__, "--phase", which, p], check=True)
            with np.load(p) as z:
                merged.update({k: z[k] for k in z.files})
    # parts of under 1 MB each (tests/_golden_check.load merges them), largest arrays first
    import io

    def size(d):
        b = io.BytesIO()
        np.savez_compressed(b, **d)
        return b.tell()

    parts, cur = [], {}
    for k in sorted(merged, key=lambda k: -merged[k].nbytes):
        trial = dict(cur, **{k: merged[k]})
        if cur and size(trial) > 900_000:
            parts.append(cur)
            cur = {k: merged[k]}
        else:
            cur = trial
    parts.append(cur)
    for old in HERE.glob("reference_vectors_*.npz"):
        old.unlink()
    for i, part in enumerate(parts):
        path = HERE / f"reference_vectors_{i}.npz"
        np.savez_compressed(path, **part)
        print(f"wrote {path} ({path.stat().st_size} bytes, {len(part)} arrays)")


if __name__ == "__main__":
    main()
