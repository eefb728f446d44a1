"""CPU tests of the tensor-parallel LLM.int8() layers: the row and input-feature slices of a globally quantised weight,
the sharding errors, and the argument checks of the native wrappers (against a fake library), including the 4-bit
multi-destination and partial GEMMs, and the destination order of the symmetric-memory slots."""
import pytest
import torch

import bitsandbytes_b200.backends.cuda as cb
from bitsandbytes_b200.parallel import (ColumnParallelLinear8bitLt, RowParallelLinear8bitLt, slice_int8_weight,
                                        slice_int8_weight_k)
from tests._parallel_sim import fake, simulate  # noqa: F401  (fake: a fixture)


def _weight(N=64, K=256, seed=3):
    g = torch.Generator().manual_seed(seed)
    CB = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8)
    SCB = torch.rand(N, generator=g) * 3
    return CB, SCB


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_row_slices_reassemble(world):
    CB, SCB = _weight()
    bias = torch.randn(64)
    shards = [slice_int8_weight(CB, SCB, world, r) for r in range(world)]
    assert torch.equal(torch.cat([s.CB for s in shards]), CB)
    assert torch.equal(torch.cat([s.SCB for s in shards]), SCB)
    layers = [ColumnParallelLinear8bitLt(s, 64, bias) for s in shards]
    assert torch.equal(torch.cat([L.bias_shard for L in layers]), bias)
    assert all(s.CB.is_contiguous() and s.rows == 64 // world and s.row0 == r * (64 // world)
               for r, s in enumerate(shards))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_k_slices_reassemble(world):
    CB, SCB = _weight()
    bias = torch.randn(64)
    shards = [slice_int8_weight_k(CB, SCB, world, r) for r in range(world)]
    assert torch.equal(torch.cat([s.CB for s in shards], dim=1), CB)
    assert all(torch.equal(s.SCB, SCB) for s in shards)  # the full-row absmax, replicated
    assert [s.k0 for s in shards] == [r * 256 // world for r in range(world)]
    assert all(s.CB.is_contiguous() and s.K == 256 // world and s.rows == 64 for s in shards)
    layers = [RowParallelLinear8bitLt(s, 256, bias, input_is_parallel=False) for s in shards]
    assert all(torch.equal(L.bias, bias) for L in layers)
    x = torch.randn(3, 5, 256)
    assert torch.equal(torch.cat([L.local_input(x) for L in layers], dim=1), x.reshape(15, 256))


def test_sharding_errors():
    CB, SCB = _weight(N=60, K=256)
    with pytest.raises(ValueError, match="divisible"):
        slice_int8_weight(CB, SCB, 8, 0)               # N % world
    with pytest.raises(ValueError, match="16"):
        slice_int8_weight_k(CB, SCB, 32, 0)            # 256 % (16 * 32)
    with pytest.raises(ValueError, match="16"):
        slice_int8_weight_k(*_weight(K=200), 2, 0)     # 200 % 32
    for bad in (-1, 4):
        with pytest.raises(ValueError, match="rank"):
            slice_int8_weight(*_weight(), 4, bad)
        with pytest.raises(ValueError, match="rank"):
            slice_int8_weight_k(*_weight(), 4, bad)
    layer = RowParallelLinear8bitLt(slice_int8_weight_k(*_weight(), 4, 1), 256)
    with pytest.raises(ValueError):
        layer.local_input(torch.randn(2, 256))         # the full input to a layer that takes its slice


def _gemm_args(M=8, N=32, K=64):
    CA = torch.zeros(M, K, dtype=torch.int8)
    CB = torch.zeros(N, K, dtype=torch.int8)
    return CA, CB, torch.ones(M), torch.ones(N)


def test_gemm_multi_out_checks(fake):
    CA, CB, SCA, SCB = _gemm_args()
    i32 = lambda *s: torch.zeros(*s, dtype=torch.int32)  # noqa: E731
    assert cb.int8_gemm_multi_out(CA, CB, None, None, [i32(8, 32)] * 8, 32, None)
    assert fake.names() == ["cbnb_b200_int8_gemm_multi_out"]
    with pytest.raises(ValueError, match="between 1 and 8"):
        cb.int8_gemm_multi_out(CA, CB, None, None, [i32(8, 32)] * 9, 32, None)
    with pytest.raises(ValueError, match="between 1 and 8"):
        cb.int8_gemm_multi_out(CA, CB, None, None, [], 32, None)
    with pytest.raises(ValueError, match="elements"):
        cb.int8_gemm_multi_out(CA, CB, None, None, [i32(7 * 40 + 32 - 1)], 40, None)  # room for a ragged ldc
    with pytest.raises(ValueError, match="ldc"):
        cb.int8_gemm_multi_out(CA, CB, None, None, [i32(8, 32)], 31, None)
    with pytest.raises(ValueError, match="int32"):
        cb.int8_gemm_multi_out(CA, CB, None, None, [torch.zeros(8, 32)], 32, None)
    with pytest.raises(ValueError, match="int8"):
        cb.int8_gemm_multi_out(CA.float(), CB, None, None, [i32(8, 32)], 32, None)
    with pytest.raises(ValueError, match="bias"):
        cb.int8_gemm_multi_out(CA, CB, None, None, [i32(8, 32)], 32, None, bias=torch.zeros(32))
    h = torch.zeros(8, 32, dtype=torch.float16)
    with pytest.raises(ValueError, match="SCA"):
        cb.int8_gemm_multi_out(CA, CB, SCA[:7], SCB, [h], 32, torch.float16)
    with pytest.raises(ValueError, match="bias"):
        cb.int8_gemm_multi_out(CA, CB, SCA, SCB, [h], 32, torch.float16, bias=torch.zeros(32, dtype=torch.bfloat16))
    with pytest.raises(ValueError, match="jpad"):
        cb.int8_gemm_multi_out(CA, CB, SCA, SCB, [h], 32, torch.float16, subA=torch.zeros(8, 12, dtype=torch.float16),
                               subBT=torch.zeros(32, 12, dtype=torch.float16))
    with pytest.raises(ValueError, match="together"):
        cb.int8_gemm_multi_out(CA, CB, SCA, SCB, [h], 32, torch.float16, subA=torch.zeros(8, 8, dtype=torch.float16))
    with pytest.raises(ValueError, match="dtype"):
        cb.int8_gemm_multi_out(CA, CB, SCA, SCB, [torch.zeros(8, 32)], 32, torch.float32)
    assert fake.names() == ["cbnb_b200_int8_gemm_multi_out"]


def test_reduce_and_quant_checks(fake):
    _, _, SCA, SCB = _gemm_args()
    with pytest.raises(ValueError, match="int32 CUDA"):
        cb.int8_reduce_partials(torch.zeros(2, 8, 32, dtype=torch.int32), SCA, SCB, torch.float16)  # on the CPU
    with pytest.raises(ValueError, match="int32"):
        cb.int8_reduce_partials(torch.zeros(2, 8, 32), SCA, SCB, torch.float16)
    with pytest.raises(ValueError, match="float16 or bfloat16"):
        cb.int8_row_stats(torch.zeros(4, 16), 0.0)
    with pytest.raises(ValueError, match="float16 or bfloat16"):
        cb.int8_quant_with_stats(torch.zeros(4, 16, dtype=torch.int8), torch.ones(4), 0.0)
    with pytest.raises(ValueError, match="jpad"):
        cb.int8_outlier_operands(torch.zeros(4, 64, dtype=torch.float16), torch.zeros(32, 64, dtype=torch.int8),
                                 torch.ones(32), torch.arange(5), jpad=4)
    assert fake.names() == []


def _gemm4_args(M=8, N=32, K=64, dtype=torch.bfloat16):
    """(A, B, shapeB, absmax, blocksize, quant_type) of an NF4 weight [N, K], blocksize 64."""
    return (torch.zeros(M, K, dtype=dtype), torch.zeros(N * K // 2, dtype=torch.uint8), (N, K),
            torch.ones(N * K // 64), 64, "nf4")


def test_gemm_4bit_multi_out_checks(fake):
    """The fused all-gather wrapper checks its operands and destinations as the plain GEMM does, before any native
    call; a raw address is the caller's to vouch for."""
    A, B, shapeB, absmax, bs, qt = _gemm4_args()

    def call(*, A=A, shapeB=shapeB, bs=bs, qt=qt, bias=None, outs=(0x1000, 0x2000), ldc=32):
        return cb.gemm_4bit_multi_out(A, B, shapeB, absmax, bs, qt, bias, None, None, None, list(outs), ldc)

    assert call() and call(outs=[torch.zeros(8, 32, dtype=torch.bfloat16)])
    assert fake.names() == ["cbnb_b200_gemm_4bit_multi_out"] * 2
    for kwargs, match in [({"bs": 48}, "blocksize"), ({"qt": "int4"}, "quant_type"), ({"shapeB": (32, 128)}, "inner"),
                          ({"outs": []}, "between 1 and 8"), ({"outs": [0x1000] * 9}, "between 1 and 8"),
                          ({"ldc": 31}, "ldc"), ({"bias": torch.zeros(32)}, "bias"),
                          ({"outs": [torch.zeros(8, 32)]}, "bfloat16"),
                          ({"outs": [torch.zeros(7 * 32 + 31, dtype=torch.bfloat16)]}, "elements")]:
        with pytest.raises(RuntimeError, match=match):
            call(**kwargs)
    assert not call(A=A.float())  # fp32 activations do not take the wgmma kernel: the caller falls back
    assert fake.names() == ["cbnb_b200_gemm_4bit_multi_out"] * 2


def test_destination_checks_keep_each_wrappers_exception(fake):
    """The 4-bit partial GEMM raises RuntimeError and the int8 multi-destination GEMM ValueError for the same bad
    destination lists."""
    A, B, shapeB, absmax, bs, qt = _gemm4_args()
    CA, CB, _, _ = _gemm_args()
    f32, i32 = torch.zeros(8, 32), torch.zeros(8, 32, dtype=torch.int32)
    assert cb.gemm_4bit_partial(A, B, shapeB, absmax, bs, qt, None, None, None, [f32] * 8, 32)
    assert cb.int8_gemm_multi_out(CA, CB, None, None, [i32] * 8, 32, None)
    short = 7 * 32 + 31  # one element less than an [8, 32] output needs
    for outs, ldc in [([f32] * 9, 32), ([], 32), ([f32], 31), ([torch.zeros(short)], 32), ([i32], 32)]:
        with pytest.raises(RuntimeError):
            cb.gemm_4bit_partial(A, B, shapeB, absmax, bs, qt, None, None, None, outs, ldc)
    for outs, ldc in [([i32] * 9, 32), ([], 32), ([i32], 31), ([torch.zeros(short, dtype=torch.int32)], 32), ([f32], 32)]:
        with pytest.raises(ValueError):
            cb.int8_gemm_multi_out(CA, CB, None, None, outs, ldc, None)
    assert fake.names() == ["cbnb_b200_gemm_4bit_partial", "cbnb_b200_int8_gemm_multi_out"]


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_peer_slots_list_the_own_buffer_first(monkeypatch, world):
    """For every rank of a simulated world, the destination list of a symmetric-memory slot is this rank's own buffer
    at the offset, then the peers' in rank order, and successive steps alternate between the two slots."""
    import bitsandbytes_b200.parallel as par

    for rank in range(world):
        simulate(monkeypatch, world, rank, [])
        gather = par.PeerGather(4, 16, torch.bfloat16, "cpu")
        parts = par.PeerPartials(4, 16, "cpu", dtype=torch.int32)
        assert (gather.M, gather.N, gather.dtype, gather.world, gather.rank) == (4, 16, torch.bfloat16, world, rank)
        assert (parts.M, parts.N, parts.dtype, parts.world, parts.rank) == (4, 16, torch.int32, world, rank)
        assert parts.bufs[0].shape == (world, 4, 16) and gather.bufs[0].shape == (4, 16)
        order = [rank] + [r for r in range(world) if r != rank]
        for peers, slot0 in ((gather, 0), (parts, 2)):
            for step in range(3):
                local, bases, _ = peers.slot()
                assert local is peers.bufs[step & 1]
                assert bases == [(slot0 + (step & 1) + 1) * 1_000_000 + r * 10_000 for r in range(world)]
                assert peers.dest_ptrs(bases, 96) == [bases[r] + 96 for r in order]
