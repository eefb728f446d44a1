"""GPU parity: the persistent grid of the wgmma 4-bit GEMM.  A grid has at most one CTA per SM, and each CTA runs
every gridDim-th tile with the stage ring's slot and phase carried from one tile to the next.  Problems with more
tiles than SMs make CTAs run several tiles; each is checked against the double-precision oracle and -- without a
K split, where the k16 summation order is the same -- bit for bit between the 256- and 128-token tiles."""
import pytest
import torch

from tests.test_gpu_gemm4 import assert_close_to_exact, exact, make_problem
from tests.test_gpu_gemm4_mt256 import run_tile

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K,qt,dtype,kw", [
    # 4 x 47 tiles of 5 stages each against a ring of 4 (MT = 256): the ring's slot and phase wrap in the middle of a
    # tile and carry across tiles
    (777, 6016, 320, "nf4", "bf16", {}),
    # one stage per tile
    (1000, 4352, 64, "fp4", "bf16", dict(bias=True)),
    # nested statistics, bias and fp16 over 5 x 40 tiles of 7 stages
    (1100, 5000, 448, "nf4", "fp16", dict(bs=128, nested=True, bias=True)),
])
def test_tiles_beyond_one_wave(M, N, K, qt, dtype, kw):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert -(-M // 256) * -(-N // 128) > sms, "the problem must have more 256-token tiles than SMs"
    p = make_problem(M, N, K, qt, dtype, **kw)
    y64 = exact(p)
    got = run_tile(p, 256, 1)
    assert_close_to_exact(got, y64, dtype, K)
    base = run_tile(p, 128, 1)
    assert_close_to_exact(base, y64, dtype, K)
    assert torch.equal(got.view(torch.int16), base.view(torch.int16)), "256- and 128-token tiles disagree"
