"""INTEGRATION.md section 1a, exercised: the UNMODIFIED reference Python package (baseline/_ref, installed by
tools/install_reference.sh from the reference checkout) loads ``libbitsandbytes_b200.so`` through its own
``cextension.py`` -- the library is dropped into the package directory under the name the reference's loader looks
for and selected with its ``BNB_CUDA_VERSION`` override (reference cextension.py:38-51) -- and the reference's
``functional`` / ``matmul_4bit`` / int8 ops then run on our kernels.  Their results must be bit-identical to what
our own Python layer computes from the same inputs.
"""
import os
import shutil
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent

_SCRIPT = r"""
import os, sys, torch
import bitsandbytes as bnb
import bitsandbytes.functional as F
from bitsandbytes.cextension import lib
assert type(lib).__name__ == "CudaBNBNativeLibrary", type(lib).__name__
out = {}
torch.manual_seed(0)
W = (torch.randn(512, 1024, device="cuda") / 32).to(torch.bfloat16)
q, qs = F.quantize_4bit(W, quant_type="nf4")
out["q"], out["absmax"] = q, qs.absmax
out["deq"] = F.dequantize_4bit(q, qs)
for M in (1, 8, 700):
    x = torch.randn(M, 1024, device="cuda", dtype=torch.bfloat16)
    out[f"x{M}"] = x
    out[f"y{M}"] = bnb.matmul_4bit(x, q.t(), qs)
A8 = torch.randn(64, 1024, device="cuda")
q8, st = F.quantize_blockwise(A8, blocksize=256)
out["A8"], out["q8"], out["absmax8"] = A8, q8, st.absmax
out["deq8"] = F.dequantize_blockwise(q8, st)
Ah = torch.randn(96, 1024, device="cuda", dtype=torch.float16)
Ah[:, 17] = 9.0
CA, SCA, cols = F.int8_vectorwise_quant(Ah, threshold=6.0)
CB, SCB, _ = F.int8_vectorwise_quant(W.to(torch.float16))
C = F.int8_linear_matmul(CA, CB)
out["Ah"], out["CA"], out["SCA"], out["cols"], out["CB"], out["SCB"], out["C"] = Ah, CA, SCA, cols, CB, SCB, C
out["mmdq"] = F.int8_mm_dequant(C, SCA, SCB)
torch.cuda.synchronize()
torch.save({k: v.cpu() for k, v in out.items()}, sys.argv[1])
print("REF_LAYER_OK", lib.__class__.__name__)
"""


def test_reference_python_layer_runs_on_our_library(tmp_path):
    ref_pkg = ROOT / "baseline" / "_ref" / "bitsandbytes"
    ours = ROOT / "bitsandbytes_b200" / "libbitsandbytes_b200.so"
    if not (ref_pkg / "cextension.py").exists():
        pytest.skip("reference package not installed (tools/install_reference.sh): loader path not exercised")
    site = tmp_path / "site"
    shutil.copytree(ref_pkg, site / "bitsandbytes", ignore=shutil.ignore_patterns("__pycache__"))
    shutil.copy(ours, site / "bitsandbytes" / "libbitsandbytes_cuda999.so")
    script = tmp_path / "ref_layer.py"
    script.write_text(_SCRIPT)
    dump = tmp_path / "ref_out.pt"
    env = dict(os.environ, PYTHONPATH=str(site), BNB_CUDA_VERSION="999")
    r = subprocess.run([sys.executable, str(script), str(dump)], capture_output=True, text=True, timeout=600, env=env,
                       cwd=str(tmp_path))
    assert r.returncode == 0 and "REF_LAYER_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
    ref = torch.load(dump)

    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    def same(a, b):
        a, b = a.cpu(), b.cpu()
        if a.dtype in (torch.bfloat16, torch.float16):
            return torch.equal(a.view(torch.int16), b.view(torch.int16))
        return torch.equal(a, b)

    torch.manual_seed(0)
    W = (torch.randn(512, 1024, device="cuda") / 32).to(torch.bfloat16)
    q, qs = F.quantize_4bit(W, quant_type="nf4")
    assert same(q, ref["q"]) and same(qs.absmax, ref["absmax"]) and same(F.dequantize_4bit(q, qs), ref["deq"])
    for M in (1, 8, 700):
        # The reference's Python layer picks its own route per shape (its legacy gemv symbol for one token, its
        # dequantize + cuBLAS fallback on sm_90 for most others, reference backends/cuda/ops.py:583-623, 904-916),
        # so its result and our fused GEMM's share the weights but not the fp32 summation order: the tolerance is
        # BASELINE.json's (<= 1e-3 relative for bf16 GEMM outputs); everything elementwise below is bit for bit.
        ours = bnb.matmul_4bit(ref[f"x{M}"].cuda(), q.t(), qs)
        rel = (ours.float().cpu() - ref[f"y{M}"].float()).norm() / ref[f"y{M}"].float().norm()
        assert rel.item() <= 1e-3, (M, rel.item())
    q8, st = F.quantize_blockwise(ref["A8"].cuda(), blocksize=256)
    assert same(q8, ref["q8"]) and same(st.absmax, ref["absmax8"]) and same(F.dequantize_blockwise(q8, st), ref["deq8"])
    CA, SCA, cols = F.int8_vectorwise_quant(ref["Ah"].cuda(), threshold=6.0)
    assert same(CA, ref["CA"]) and same(SCA, ref["SCA"]) and same(cols, ref["cols"])
    CB, SCB, _ = F.int8_vectorwise_quant(W.to(torch.float16))
    assert same(CB, ref["CB"]) and same(SCB, ref["SCB"])
    C = F.int8_linear_matmul(CA, CB)
    assert same(C, ref["C"]) and same(F.int8_mm_dequant(C, SCA, SCB), ref["mmdq"])
