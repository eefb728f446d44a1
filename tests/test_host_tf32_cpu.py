"""CPU: the host picks the native dtype of an fp32 4-bit GEMM from PyTorch's fp32 matmul precision -- 3 (TF32
tensor cores) for every way PyTorch offers of allowing TF32, 0 (the fp32 CUDA-core route) otherwise.  Each case runs
in a fresh interpreter: once the legacy and the per-backend precision APIs have been mixed, torch's legacy getters
raise for the rest of the process."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]

CASES = [
    ("", 0),
    ("torch.backends.cuda.matmul.allow_tf32 = True", 3),
    ("torch.backends.cuda.matmul.allow_tf32 = False", 0),
    ("torch.set_float32_matmul_precision('high')", 3),
    ("torch.set_float32_matmul_precision('medium')", 3),
    ("torch.set_float32_matmul_precision('highest')", 0),
    ("torch.backends.cuda.matmul.fp32_precision = 'tf32'", 3),
    ("torch.backends.cuda.matmul.fp32_precision = 'ieee'", 0),
    ("torch.backends.fp32_precision = 'tf32'", 3),  # inherited by the matmul backend
    ("torch.backends.fp32_precision = 'tf32'; torch.backends.cuda.matmul.fp32_precision = 'ieee'", 0),
    ("torch.backends.cuda.matmul.allow_tf32 = True; torch.backends.cuda.matmul.fp32_precision = 'ieee'", 0),
    ("torch.set_float32_matmul_precision('high'); torch.backends.cuda.matmul.fp32_precision = 'tf32'", 3),
]


@pytest.mark.parametrize("setting,want", CASES)
def test_fp32_dtype_follows_the_matmul_precision(setting, want):
    code = (
        "import warnings; warnings.simplefilter('ignore')\n"
        "import torch\n"
        f"{setting}\n"
        "from bitsandbytes_b200.backends.cuda import gemm_4bit_dtype_id\n"
        "print(gemm_4bit_dtype_id(torch.float32), gemm_4bit_dtype_id(torch.float16), gemm_4bit_dtype_id(torch.bfloat16))\n"
    )
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split()[-3:] == [str(want), "1", "2"]


def test_path_query_for_tf32():
    """Which kernel a dtype-3 GEMM takes is a pure function of the shape: the wgmma GEMM from 4 tokens on (the
    measured crossover) where it serves the shape, the fp32 route otherwise; dtype 0 is unchanged."""
    from bitsandbytes_b200 import cextension

    path = cextension.lib.cbnb_b200_gemm_4bit_path
    for M in (4, 5, 8, 9, 16, 4096):
        assert path(M, 4096, 4096, 64, 3) == 1
        assert path(M, 4096, 4096, 64, 0) == 2
    for M in range(1, 4):
        assert path(M, 4096, 4096, 64, 3) == 2
    assert path(4096, 4096, 4000, 64, 3) == 2    # K % 64 != 0
    assert path(4096, 4096, 4096, 48, 3) == 2    # blocksize not a power of two
