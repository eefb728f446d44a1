"""GPU parity: the wgmma 4-bit GEMM at its 256-token tile (64-deep stages, one table per row and block) through the
developer entry, against the double-precision oracle and -- without a K split, where the k16 summation order is the
same -- bit for bit against the 128-token tile."""
import pytest
import torch

from tests import _native as nat
from tests.test_gpu_gemm4 import assert_close_to_exact, exact, make_problem

pytestmark = pytest.mark.gpu


def run_tile(p, mt, splits):
    M, N, K = p["M"], p["N"], p["K"]
    out = torch.full((M, N), float("nan"), device="cuda", dtype=nat.DTYPE[p["dtype"]])
    rc = nat.lib.cbnb_b200_gemm_4bit_pair(
        nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
        nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]), nat.ptr(out), nat.ptr(p["bias"]), M, N, K, N, p["bs"],
        nat.QT_ID[p["qt"]], nat.DTYPE_ID[p["dtype"]], mt, splits, None, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0, (mt, splits)
    return out


# K = 576 and 448 are multiples of 64 but not of 128: the 128-token tile ends on a half stage, and at blocksize 128
# every odd row starts in the middle of a quantisation block
@pytest.mark.parametrize("M,N,K,qt,dtype,kw", [
    (600, 328, 448, "nf4", "bf16", {}),
    (513, 256, 576, "fp4", "fp16", dict(bias=True)),
    (300, 200, 576, "nf4", "bf16", dict(bs=128, nested=True, bias=True)),
    (777, 384, 320, "nf4", "fp16", dict(bs=32, nested=True)),
    (256, 130, 1024, "fp4", "bf16", dict(bs=32, bias=True)),
])
def test_mt256_vs_oracle_and_mt128(M, N, K, qt, dtype, kw):
    p = make_problem(M, N, K, qt, dtype, **kw)
    y64 = exact(p)
    got = run_tile(p, 256, 1)
    assert_close_to_exact(got, y64, dtype, K)
    base = run_tile(p, 128, 1)
    assert torch.equal(got.view(torch.int16), base.view(torch.int16)), "256- and 128-token tiles disagree"
    # a forced K split: every split's partial tile goes through the workspace and the split-order reduction
    split = run_tile(p, 256, 3)
    assert_close_to_exact(split, y64, dtype, K)
