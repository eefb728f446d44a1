"""Host side of the row-parallel (input-feature-sharded) Linear4bit: slicing a globally quantised weight by K, the
nested statistics turned into plain fp32 scales, and the shape rules (bitsandbytes_b200/parallel.py)."""
import numpy as np
import pytest
import torch

import oracle


def _problem(N=256, K=1024, bs=64, qt="nf4", seed=11):
    g = torch.Generator().manual_seed(seed)
    W = (torch.randn(N, K, generator=g) / K**0.5).to(torch.bfloat16)
    packed, absmax = oracle.quantize_blockwise(W.float().numpy().reshape(-1), bs, qt)
    return N, K, torch.from_numpy(packed), torch.from_numpy(absmax)


def _state(absmax, N, K, bs, qt, nested):
    import bitsandbytes_b200.functional as F

    if not nested:
        return F.QuantState(absmax=absmax, shape=torch.Size([N, K]), code=None, blocksize=bs, quant_type=qt,
                            dtype=torch.bfloat16)
    offset = absmax.mean()
    code2 = F.create_dynamic_map()
    a8, a2 = oracle.quantize_blockwise((absmax - offset).numpy(), 256, None, code2.numpy())
    s2 = F.QuantState(absmax=torch.from_numpy(a2), code=code2, blocksize=256, dtype=torch.float32)
    return F.QuantState(absmax=torch.from_numpy(a8), shape=torch.Size([N, K]), code=F.get_4bit_type(qt, "cpu"),
                        blocksize=bs, quant_type=qt, dtype=torch.bfloat16, offset=offset, state2=s2)


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("bs", [32, 64, 128])
def test_k_slices_reassemble_the_global_weight(world, bs):
    """The K shards, put side by side, are the global packed weight and absmax byte for byte."""
    from bitsandbytes_b200.parallel import slice_quantized_weight_k

    N, K, packed, absmax = _problem(bs=bs)
    qs = _state(absmax, N, K, bs, "nf4", nested=False)
    shards = [slice_quantized_weight_k(packed, qs, world, r) for r in range(world)]
    for r, s in enumerate(shards):
        assert (s.rows, s.K, s.k0, s.blocksize) == (N, K // world, r * K // world, bs)
        assert s.absmax_8bit is None and s.packed.is_contiguous() and s.absmax.is_contiguous()
    codes = torch.cat([s.packed.view(N, -1) for s in shards], dim=1)
    scales = torch.cat([s.absmax.view(N, -1) for s in shards], dim=1)
    assert torch.equal(codes.reshape(-1), packed)
    assert torch.equal(scales.reshape(-1).view(torch.int32), absmax.view(torch.int32))


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("qt", ["nf4", "fp4"])
def test_nested_shards_carry_the_double_quant_scales(world, qt):
    """A nested state's shards hold plain fp32 scales equal to the oracle's double-quant scales, and decode to the
    same weights as the global tensor's columns, bit for bit."""
    from bitsandbytes_b200.parallel import nested_scales, slice_quantized_weight_k

    N, K, packed, absmax = _problem(qt=qt, bs=64)
    qs = _state(absmax, N, K, 64, qt, nested=True)
    want = oracle.nested_absmax(qs.state2.absmax.numpy(), qs.absmax.numpy(), qs.state2.code.numpy(), float(qs.offset))
    assert np.array_equal(nested_scales(qs).numpy().view(np.uint32), want.view(np.uint32))
    full = oracle.dequantize_blockwise(packed.numpy(), want, 64, N * K, qt, None, "bf16").reshape(N, K)
    kr = K // world
    for r in range(world):
        s = slice_quantized_weight_k(packed, qs, world, r)
        assert s.absmax_8bit is None and s.absmax.dtype == torch.float32
        assert np.array_equal(s.absmax.numpy().reshape(N, -1), want.reshape(N, -1)[:, r * kr // 64:(r + 1) * kr // 64])
        part = oracle.dequantize_blockwise(s.packed.numpy(), s.absmax.numpy(), 64, N * kr, qt, None, "bf16")
        assert np.array_equal(part.reshape(N, kr), full[:, r * kr:(r + 1) * kr])


def test_bad_k_raises():
    from bitsandbytes_b200.parallel import slice_quantized_weight_k

    N, K, packed, absmax = _problem(K=1024, bs=64)
    qs = _state(absmax, N, K, 64, "nf4", nested=False)
    with pytest.raises(ValueError):
        slice_quantized_weight_k(packed, qs, 3, 0)          # 1024 % (3 * 64)
    with pytest.raises(ValueError):
        slice_quantized_weight_k(packed, qs, 32, 0)         # 1024 % (32 * 64)
    N, K, packed, absmax = _problem(K=1024, bs=32)
    qs = _state(absmax, N, K, 32, "nf4", nested=False)
    with pytest.raises(ValueError):
        slice_quantized_weight_k(packed, qs, 32, 0)         # 32 features per shard: not a multiple of 64
    with pytest.raises(ValueError):
        slice_quantized_weight_k(packed, qs, 2, 2)          # no rank 2 in a world of 2


def test_row_parallel_input_slicing():
    """The layer takes its own x_r, or slices the full x at its k0, and rejects other widths."""
    from bitsandbytes_b200.parallel import RowParallelLinear4bit, slice_quantized_weight_k

    N, K, packed, absmax = _problem(K=1024, bs=64)
    qs = _state(absmax, N, K, 64, "nf4", nested=False)
    x = torch.randn(3, 5, K)
    full = RowParallelLinear4bit(slice_quantized_weight_k(packed, qs, 4, 2), K, input_is_parallel=False)
    assert torch.equal(full.local_input(x), x[..., 512:768])
    own = RowParallelLinear4bit(slice_quantized_weight_k(packed, qs, 4, 2), K)
    assert torch.equal(own.local_input(x[..., :256]), x[..., :256])
    with pytest.raises(ValueError):
        own.local_input(x)
    with pytest.raises(ValueError):
        full.local_input(x[..., :256])
