"""CPU: the grouped LLM.int8() GEMM's op schema and shape function, its argument checks (each refusal before any native
call), the native calls it makes (recorded by a stand-in library), the autograd refusals and GroupedLinear8bitLt before
quantisation and through a state-dict round trip."""
import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.backends.cuda as cb
from bitsandbytes_b200 import _ops  # noqa: F401  (defines the ops)
from tests._parallel_sim import install_fake_lib

BF = torch.bfloat16


def _args(E=4, N=192, K=256, M=50, dtype=BF, device="meta"):
    return dict(A=torch.empty(M, K, dtype=dtype, device=device), CB=torch.empty(E, N, K, dtype=torch.int8, device=device),
                SCB=torch.empty(E * N, device=device), offs=torch.empty(E, dtype=torch.int32, device=device))


def _call(**kw):
    return torch.ops.bitsandbytes.int8_grouped_mm(**kw)


def test_schema_and_shape_function():
    op = torch.ops.bitsandbytes.int8_grouped_mm.default
    assert [a.name for a in op._schema.arguments] == ["A", "CB", "SCB", "offs", "threshold", "bias"]
    for dtype in (torch.float16, BF):
        out = _call(**_args(dtype=dtype), threshold=6.0, bias=torch.empty(4, 192, dtype=dtype, device="meta"))
        assert out.shape == (50, 192) and out.dtype == dtype and out.device.type == "meta"
    assert _call(**_args(M=0)).shape == (0, 192)
    assert _call(**_args(E=1024, N=8, K=16)).shape == (50, 8)


def test_shape_function_under_fake_tensor_mode():
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        out = _call(**_args(device="cpu"), threshold=6.0)
    assert tuple(out.shape) == (50, 192) and out.dtype == BF


# each refusal of the contract with its message
REFUSALS = [
    (dict(A=torch.empty(50, 256)), "A must be float16 or bfloat16"),                                # fp32 activations
    (dict(A=torch.empty(50, 200, dtype=BF), CB=torch.empty(4, 192, 200, dtype=torch.int8)), "multiple of 16"),
    (dict(CB=torch.empty(1025, 8, 256, dtype=torch.int8), SCB=torch.empty(1025 * 8),
          offs=torch.empty(1025, dtype=torch.int32)), "1 <= E <= 1024"),                            # E > 1024
    (dict(CB=torch.empty(4 * 192, 256, dtype=torch.int8)), r"\[E, N, K\] expert tensor"),           # a 2-D weight
    (dict(CB=torch.empty(4, 192, 256, dtype=torch.uint8)), r"int8 \[E, N, K\]"),
    (dict(SCB=torch.empty(192)), r"SCB must be float32 \[768\]"),                                  # SCB size
    (dict(SCB=torch.empty(4, 192)), r"SCB must be float32 \[768\]"),
    (dict(SCB=torch.empty(768, dtype=torch.float16)), r"SCB must be float32"),
    (dict(offs=torch.empty(4, dtype=torch.int64)), "offs must be int32"),
    (dict(offs=torch.empty(5, dtype=torch.int32)), "offs must be int32"),
    (dict(A=torch.empty(50, 192, dtype=BF)), r"A must be \[M, 256\]"),
    (dict(bias=torch.empty(4 * 192, dtype=BF)), r"bias must be torch.bfloat16 \[4, 192\]"),        # bias shape
    (dict(bias=torch.empty(4, 192, dtype=torch.float16)), r"bias must be torch.bfloat16"),          # bias dtype
    (dict(threshold=-1.0), "non-negative"),
]


@pytest.mark.parametrize("change,match", REFUSALS)
def test_refusals_before_any_native_call(monkeypatch, change, match):
    lib = install_fake_lib(monkeypatch)
    kw = _args(device="cpu")
    kw.update(change)
    with pytest.raises(RuntimeError, match=match):
        cb.int8_grouped_mm(**kw)
    with pytest.raises(RuntimeError, match=match):  # the shape function makes the same checks
        _call(**{k: (v.to("meta") if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    assert lib.calls == []


@pytest.mark.parametrize("threshold", [0.0, 6.0])
@pytest.mark.parametrize("dtype,bias", [(torch.float16, False), (BF, True)])
def test_native_calls(monkeypatch, threshold, dtype, bias):
    """The activations are quantised as fp16 without the global flags, the per-expert outliers are prepared only with a
    threshold, and the GEMM gets the stacked weights, the offsets and (with a threshold) the outlier operands."""
    lib = install_fake_lib(monkeypatch)
    E, N, K, M = 4, 192, 256, 50
    kw = _args(E, N, K, M, dtype=dtype, device="cpu")
    b = torch.zeros(E, N, dtype=dtype) if bias else None
    out = cb.int8_grouped_mm(**kw, threshold=threshold, bias=b)
    assert out.shape == (M, N) and out.dtype == dtype
    names = lib.names()
    want = ["cbnb_b200_int8_vector_quant_flags"] + (["cbnb_b200_int8_grouped_outliers"] if threshold else []) + \
        ["cbnb_b200_int8_grouped_mm"]
    assert names == want
    q = lib.calls[0][1]
    assert q[3] is None and q[4] == threshold and q[5:8] == (M, K, 1)  # no global flags; rows, cols, fp16
    if dtype == torch.float16:
        assert q[0] == kw["A"].data_ptr()  # fp16 activations are quantised in place, not copied
    g = lib.calls[-1][1]
    assert g[1] == kw["CB"].data_ptr() and g[3] == kw["SCB"].data_ptr() and g[5] == kw["offs"].data_ptr()
    assert g[6] == E and g[13:17] == (M, N, K, 1 if dtype == torch.float16 else 2)
    assert (g[4] is not None) == bias
    if threshold:
        o = lib.calls[1][1]
        assert o[6] == E and o[7] == threshold and o[14:18] == g[13:17]
        assert o[2] == g[0]                            # CA: zeroed by the preparation, read by the GEMM
        assert o[10:14] == (g[10], g[11], g[8], g[9])  # cols, count, subA, subBT
        assert g[7] == kw["A"].data_ptr()              # the columns past 64 are gathered from A
    else:
        assert g[7:12] == (None,) * 5
    lib.calls.clear()
    assert cb.int8_grouped_mm(**_args(M=0, device="cpu"), threshold=threshold).shape == (0, 192)
    assert lib.calls == []


def test_a_refused_launch_raises(monkeypatch):
    lib = install_fake_lib(monkeypatch)
    lib.refuse.add("cbnb_b200_int8_grouped_mm")
    with pytest.raises(RuntimeError, match="does not serve this call"):
        cb.int8_grouped_mm(**_args(device="cpu"))


def test_grouped_matmul_8bit_refusals():
    kw = _args(device="cpu")
    A = kw["A"].requires_grad_(True)
    with pytest.raises(ValueError, match="bfloat16 only"):
        bnb.grouped_matmul_8bit(A.detach().half().requires_grad_(True), kw["CB"], kw["SCB"], kw["offs"])
    with pytest.raises(ValueError, match="N % 8"):
        bnb.grouped_matmul_8bit(A, torch.empty(4, 190, 256, dtype=torch.int8), torch.empty(4 * 190), kw["offs"])
    with pytest.raises(RuntimeError, match=r"\[E, N, K\] expert tensor"):
        bnb.grouped_matmul_8bit(A, torch.empty(768, 256, dtype=torch.int8), kw["SCB"], kw["offs"])


def test_grouped_linear8bitlt_before_quantisation():
    from bitsandbytes_b200.nn import GroupedLinear8bitLt, Int8Params, Linear8bitLt

    m = GroupedLinear8bitLt(8, 256, 192, bias=True, threshold=6.0)
    assert isinstance(m.weight, Int8Params) and m.weight.dtype == torch.float32 and not m.weight.has_fp16_weights
    assert m.weight.shape == (8, 192, 256) and m.bias.shape == (8, 192) and not m.weight.requires_grad
    assert set(m.state_dict()) == {"weight", "bias"} == set(Linear8bitLt(256, 192, bias=True).state_dict())
    assert set(GroupedLinear8bitLt(2, 64, 64).state_dict()) == {"weight"}
    assert "num_experts=8" in repr(m) and "threshold=6.0" in repr(m)
    assert m.weight.abs().max().item() <= 256**-0.5 + 1e-6
    with pytest.raises(ValueError, match="has_fp16_weights"):
        GroupedLinear8bitLt(8, 256, 192, has_fp16_weights=True)
    with pytest.raises(RuntimeError, match="not quantised"):
        m(torch.empty(4, 256, dtype=BF), torch.zeros(8, dtype=torch.int32))


def test_state_dict_loads_quantised_codes_before_cuda():
    """A quantised checkpoint (Linear8bitLt's keys) loads into a module that has not been moved to CUDA yet."""
    from bitsandbytes_b200.nn import GroupedLinear8bitLt

    E, N, K = 3, 16, 32
    sd = {"weight": torch.randint(-127, 128, (E, N, K), dtype=torch.int8), "SCB": torch.rand(E * N) + 0.5,
          "weight_format": torch.tensor(0, dtype=torch.uint8), "bias": torch.randn(E, N)}
    m = GroupedLinear8bitLt(E, K, N, bias=True)
    m.load_state_dict(sd)
    assert m.weight.dtype == torch.int8 and torch.equal(m.weight.data, sd["weight"])
    assert torch.equal(m.weight.SCB, sd["SCB"]) and torch.equal(m.bias.data, sd["bias"])
    out = m.state_dict()
    assert set(out) == {"weight", "SCB", "weight_format", "bias"}
    assert torch.equal(out["weight"], sd["weight"]) and torch.equal(out["SCB"], sd["SCB"])
    with pytest.raises(RuntimeError, match="size mismatch"):
        GroupedLinear8bitLt(E, K, N + 8, bias=True).load_state_dict(sd)
