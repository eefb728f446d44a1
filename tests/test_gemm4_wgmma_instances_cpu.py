"""CPU: the case table of test_gpu_gemm4_wgmma_instances covers every non-grouped instance of the fused wgmma 4-bit
GEMM, with a K split at every token tile that can split, on an H100 SXM (132 SMs) and an H100 PCIe (114 SMs) alike.
Building the table also checks that every dispatched shape takes its intended tile and split by the restated rule."""
from itertools import product

import pytest

from tests.test_gpu_gemm4_wgmma_instances import (DQS, DT16, QTS, TILES16, TILES_TF32, all_cases, dispatched_shape,
                                                  expected, instance, split_of, tile_rule)

SMS = [132, 114]


def _runs(sms):
    return [r for c in all_cases(sms) for r in expected(c, sms)]


@pytest.mark.parametrize("sms", SMS)
def test_the_case_table_covers_all_112_instances(sms):
    want = {instance(dt, qt, mt, dq, part) for dt, qt, mt, dq, part in product(DT16, QTS, TILES16, DQS, (0, 1))}
    want |= {instance("tf32", qt, mt, dq, part) for qt, mt, dq, part in product(QTS, TILES_TF32, DQS, (0, 1))}
    assert len(want) == 112
    assert {i for i, _ in _runs(sms)} == want


@pytest.mark.parametrize("sms", SMS)
def test_every_tile_up_to_128_has_a_split_case(sms):
    split = {(i[1], i[3], i[5]) for i, s in _runs(sms) if s > 1}
    for t, mt, part in product(["__nv_bfloat16", "__half", "float"], TILES_TF32, "01"):
        assert (t, str(mt), part) in split, (t, mt, part)


@pytest.mark.parametrize("sms", SMS)
def test_dispatched_shapes_follow_the_rule(sms):
    for dt, mt, split in product(DT16 + ["tf32"], TILES16, [False, True]):
        if mt == 256 and (split or dt == "tf32"):
            continue
        M, N, K = dispatched_shape(mt, split, dt, sms)
        assert tile_rule(M, N, dt, sms) == mt
        assert (split_of(M, N, K, mt, dt, sms)[0] > 1) == split


def test_the_restated_split_rule():
    # 2 tiles on 132 SMs: 66 by the grid, at most kb / 2 = 4 of 9 stages -> 3 stages per split, 3 splits
    assert split_of(15, 203, 1152, 16, "bf16", 132) == (3, 3)
    assert split_of(15, 203, 1152, 16, "tf32", 132) == (9, 2)  # 64-deep fp32 stages
    assert split_of(100, 203, 640, 16, "bf16", 132, force=3) == (3, 2)  # 2, 2, 1 k-blocks
    assert split_of(100, 203, 640, 256, "fp16", 132, force=3) == (3, 4)  # 4, 4, 2
    assert split_of(150, 203, 2048, 16, "bf16", 132, force=8) is None  # 20 tiles x 8 splits > one wave
    assert split_of(1000, 4187, 320, 256, "bf16", 132) == (1, 5)
