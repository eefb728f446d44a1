"""CPU: the grouped 4-bit GEMM's op schema and shape function, its argument checks and GroupedLinear4bit before
quantisation.  The op runs on meta tensors here: its shape function is the host-side check the CUDA kernel also runs."""
import pytest
import torch

import bitsandbytes_b200 as bnb
from bitsandbytes_b200 import _ops  # noqa: F401  (defines the ops)
from bitsandbytes_b200.functional import QuantState


def _args(E=4, N=192, K=256, M=50, bs=64, dtype=torch.bfloat16, nested=False, device="meta"):
    n = E * N * K
    nb = -(n // -bs)
    kw = dict(A=torch.empty(M, K, dtype=dtype, device=device), B=torch.empty(n // 2, 1, dtype=torch.uint8, device=device),
              shapeB=[E, N, K], absmax=torch.empty(nb, device=device), blocksize=bs, quant_type="nf4",
              offs=torch.empty(E, dtype=torch.int32, device=device))
    if nested:
        kw.update(absmax=torch.empty(-(nb // -256), device=device), absmax_8bit=torch.empty(nb, dtype=torch.uint8,
                  device=device), absmax_code=torch.empty(256, device=device),
                  absmax_offset=torch.empty((), device=device))
    return kw


def _call(**kw):
    return torch.ops.bitsandbytes.gemm_4bit_grouped(**kw)


def test_schema_and_shape_function():
    op = torch.ops.bitsandbytes.gemm_4bit_grouped.default
    assert [a.name for a in op._schema.arguments] == ["A", "B", "shapeB", "absmax", "blocksize", "quant_type", "offs",
                                                       "bias", "absmax_8bit", "absmax_code", "absmax_offset"]
    for nested in (False, True):
        out = _call(**_args(nested=nested))
        assert out.shape == (50, 192) and out.dtype == torch.bfloat16 and out.device.type == "meta"
    kw = _args(dtype=torch.float16)
    out = _call(**kw, bias=torch.empty(4, 192, dtype=torch.float16, device="meta"))
    assert out.shape == (50, 192) and out.dtype == torch.float16
    assert _call(**_args(M=0)).shape == (0, 192)


def test_shape_function_under_fake_tensor_mode():
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        out = _call(**_args(device="cpu"))
    assert tuple(out.shape) == (50, 192) and out.dtype == torch.bfloat16


@pytest.mark.parametrize("change,match", [
    (dict(shapeB=[4 * 192, 256]), r"\[E, N, K\] expert tensor"),
    (dict(offs=torch.empty(4, dtype=torch.int64, device="meta")), "offs must be int32"),
    (dict(offs=torch.empty(5, dtype=torch.int32, device="meta")), "offs must be int32"),
    (dict(A=torch.empty(50, 256, dtype=torch.float32, device="meta")), "float16 or bfloat16"),
    (dict(B=torch.empty(4 * 192 * 256 // 2 - 1, 1, dtype=torch.uint8, device="meta")), "bytes"),
    (dict(A=torch.empty(50, 192, dtype=torch.bfloat16, device="meta")), r"\[E, K, N\]"),
    (dict(absmax=torch.empty(7, device="meta")), "scales"),
    (dict(bias=torch.empty(4 * 192, dtype=torch.bfloat16, device="meta")), "bias must be"),
])
def test_argument_errors(change, match):
    kw = _args()
    kw.update(change)
    with pytest.raises(RuntimeError, match=match):
        _call(**kw)


def test_k_and_expert_limits():
    with pytest.raises(RuntimeError, match="multiple of 64"):
        _call(**_args(K=96))
    with pytest.raises(RuntimeError, match="1 <= E <= 1024"):
        _call(**_args(E=1025, N=8, K=64))
    assert _call(**_args(E=1024, N=8, K=64)).shape == (50, 8)


def test_grouped_matmul_refuses_2d_and_transposed_weights():
    qs2 = QuantState(absmax=torch.empty(1), shape=torch.Size([192, 256]), blocksize=64, quant_type="nf4",
                     dtype=torch.bfloat16)
    A = torch.empty(8, 256, dtype=torch.bfloat16)
    offs = torch.zeros(4, dtype=torch.int32)
    with pytest.raises(ValueError, match=r"\[E, N, K\]"):
        bnb.grouped_matmul_4bit(A, torch.empty(1, dtype=torch.uint8), qs2, offs)
    qs_t = QuantState(absmax=torch.empty(1), shape=torch.Size([4, 256, 192]), blocksize=64, quant_type="nf4",
                      dtype=torch.bfloat16)
    with pytest.raises(ValueError, match=r"quantise it as \[E, N, K\]"):
        bnb.grouped_matmul_4bit(A, torch.empty(1, dtype=torch.uint8), qs_t, offs)


def test_grouped_linear4bit_before_quantisation():
    from bitsandbytes_b200.nn import GroupedLinear4bit, Linear4bit, Params4bit

    m = GroupedLinear4bit(8, 256, 192, bias=True, quant_type="nf4")
    assert isinstance(m.weight, Params4bit) and not m.weight.bnb_quantized
    assert m.weight.shape == (8, 192, 256) and m.bias.shape == (8, 192)
    assert m.weight.quant_type == "nf4" and m.weight.compress_statistics and m.weight.module is m
    assert set(m.state_dict()) == {"weight", "bias"} == set(Linear4bit(256, 192, bias=True).state_dict())
    assert set(GroupedLinear4bit(2, 64, 64).state_dict()) == {"weight"}
    assert "num_experts=8" in repr(m)
    # each expert is initialised as nn.Linear initialises its weight: |w| <= 1/sqrt(in_features)
    assert m.weight.abs().max().item() <= 256**-0.5 + 1e-6
