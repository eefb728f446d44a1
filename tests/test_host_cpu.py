"""CPU-only tests (no compute calls into the CUDA library): the C-ABI surface, host logic,
serialisation formats, shape functions, the loud failure without a GPU, and the sharding
logic of the N > 1 path (world_size-2 gloo)."""
import ctypes as ct
import os
import pickle
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


# ------------------------------------------------------------------------------------ C ABI
def _declared_symbols():
    text = (ROOT / "include" / "bitsandbytes_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = re.findall(r"^\s*(?:const\s+)?[A-Za-z_][\w\s\*]*?\b(\w+)\s*\([^;{]*\)\s*;", text, flags=re.M)
    return sorted(set(n for n in names if n not in ("defined",)))


def test_library_loads_and_exports_every_declared_symbol():
    from bitsandbytes_b200 import cextension

    assert isinstance(cextension.lib, cextension.NativeLibrary), "libbitsandbytes_b200.so missing: run build()"
    dll = ct.CDLL(str(cextension.library_path()))
    declared = _declared_symbols()
    assert len(declared) >= 40, declared
    missing = [n for n in declared if not hasattr(dll, n)]
    assert not missing, f"declared in include/bitsandbytes_b200.h but not exported: {missing}"
    # and the Python signature table covers the hot-path symbols
    table = set(cextension.EXPORTED_SYMBOLS)
    for n in declared:
        if n.startswith(("cigemmlt_8",)):
            continue
        assert n in table, f"{n} has no ctypes signature in cextension.py"
    assert "sm_90a" in cextension.lib.build_info()


def test_reference_abi_names_present():
    """Every symbol the reference's CUDA backend binds for this path (reference
    bitsandbytes/backends/cuda/ops.py:16-66, cextension.py:112-115) resolves in our library."""
    from bitsandbytes_b200 import cextension

    dll = ct.CDLL(str(cextension.library_path()))
    names = [f"cdequantize_blockwise_{d}{q}" for d in ("fp32", "bf16", "fp16") for q in ("", "_nf4", "_fp4")]
    names += [f"cquantize_blockwise_{d}{q}" for d in ("fp32", "bf16", "fp16") for q in ("", "_nf4", "_fp4")]
    names += [f"cgemm_4bit_{d}" for d in ("bf16", "fp16", "fp32")]
    names += [f"cgemm_4bit_inference_naive_{d}" for d in ("bf16", "fp16", "fp32")]
    names += ["cigemmlt_32", "cdequant_mm_int32_fp16", "cint8_vector_quant", "get_context", "cget_managed_ptr",
              "cprefetch", "cigemmlt_8", "cigemmlt_8_rowscale"]
    assert not [n for n in names if not hasattr(dll, n)]


def test_entry_points_validate_arguments_before_touching_the_device():
    """Argument errors are reported through the error flag without a CUDA call (so this runs on a CPU box)."""
    from bitsandbytes_b200 import cextension

    lib = cextension.lib
    rc = lib.cbnb_b200_gemm_4bit_multi_out(None, None, None, None, None, None, None, 0, None, 16, 128, 64, 128, 64, 2, 2,
                                           None)
    assert rc == 1
    with pytest.raises(RuntimeError, match="n_outs"):
        lib.check("gemm_4bit_multi_out")
    # nine destinations is one too many (the kernel carries the local buffer + 7 peers)
    arr = (ct.c_void_p * 9)(*([0] * 9))
    rc = lib.cbnb_b200_gemm_4bit_multi_out(None, None, None, None, None, None, ct.cast(arr, ct.c_void_p), 9, None, 16,
                                           128, 64, 128, 64, 2, 2, None)
    assert rc == 1
    with pytest.raises(RuntimeError):
        lib.check("gemm_4bit_multi_out")
    # an empty problem is a no-op, and which kernel a shape would take is a pure function of the shape
    assert lib.cbnb_b200_gemm_4bit_multi_out(None, None, None, None, None, None, ct.cast(arr, ct.c_void_p), 2, None, 0,
                                             128, 64, 128, 64, 2, 2, None) == 0
    path = lib.cbnb_b200_gemm_4bit_path
    assert path(1, 4096, 4096, 64, 2) == 0      # CUDA-core GEMV
    assert path(4, 4096, 4096, 64, 2) == 3      # mma.sync decode kernel
    assert path(8, 4096, 4096, 64, 1) == 3
    assert path(9, 4096, 4096, 64, 2) == 1      # wgmma GEMM
    assert path(4096, 4096, 4096, 64, 2) == 1
    assert path(4, 4096, 4096, 64, 0) == 2      # fp32 activations: generic CUDA-core kernel
    assert path(4, 4096, 4000, 64, 2) == 2      # K % 64 != 0


def test_missing_library_fails_loudly(tmp_path):
    code = ("import os; os.environ['BNB_B200_LIBRARY']=r'%s/nope.so'\n"
            "import bitsandbytes_b200.cextension as c\n"
            "try:\n    c.lib.cquantize_blockwise_fp32\nexcept RuntimeError as e:\n    print('RAISED', e)\n") % tmp_path
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    assert "RAISED" in out.stdout and "no CPU or PyTorch fallback" in out.stdout, out.stdout + out.stderr


def test_no_cpu_fallback_for_ops():
    import bitsandbytes_b200.functional as F

    with pytest.raises(NotImplementedError):
        F.quantize_4bit(torch.randn(64, 64), quant_type="nf4")
    with pytest.raises(NotImplementedError):
        F.quantize_blockwise(torch.randn(4096))


def test_product_never_imports_the_oracle():
    for p in (ROOT / "bitsandbytes_b200").rglob("*.py"):
        src = p.read_text()
        assert "import oracle" not in src and "from oracle" not in src, p


# ------------------------------------------------------------------------------------ code books / QuantState
def test_codebooks_match_reference_golden(golden):
    import bitsandbytes_b200.functional as F

    assert np.array_equal(F.create_dynamic_map().numpy().view(np.uint32), golden["dynamic_map"].view(np.uint32))
    for q in ("nf4", "fp4"):
        assert np.array_equal(F.get_4bit_type(q, device="cpu").numpy().view(np.uint32),
                              golden[f"{q}_code"].view(np.uint32))
    m = F.create_dynamic_map(signed=False)
    assert m.numel() == 256 and m.min() == 0 and m.max() == 1


def test_nf4_tree_pivots_are_code_midpoints():
    """The decision-tree pivots of the quantiser (reference tests/test_functional.py:1037-1049
    regenerates them from the code book) are the midpoints of adjacent NF4 values."""
    import bitsandbytes_b200.functional as F

    code = F.get_4bit_type("nf4", device="cpu").double()
    mids = ((code[:-1] + code[1:]) / 2).float()
    src = (ROOT / "bitsandbytes_b200" / "csrc" / "blockwise.cu").read_text()
    body = src[src.index("quantize_nf4(float x)"):src.index("quantize_fp4(float x)")]
    lits = sorted(float(v) for v in re.findall(r"x > (-?\d\.\d+)f", body))
    assert len(lits) == 15
    assert np.allclose(np.array(lits, np.float32), np.sort(mids.numpy()), rtol=0, atol=1e-7)


def _state(nested: bool):
    import bitsandbytes_b200.functional as F

    absmax = torch.rand(64) + 0.1
    code = F.get_4bit_type("nf4", device="cpu")
    if not nested:
        return F.QuantState(absmax=absmax, shape=torch.Size([64, 64]), code=code, blocksize=64, quant_type="nf4",
                            dtype=torch.bfloat16)
    s2 = F.QuantState(absmax=torch.rand(1) + 0.1, code=F.create_dynamic_map(), blocksize=256, dtype=torch.float32)
    return F.QuantState(absmax=torch.randint(0, 256, (64,), dtype=torch.uint8), shape=torch.Size([64, 64]), code=code,
                        blocksize=64, quant_type="nf4", dtype=torch.float16, offset=torch.tensor(0.25), state2=s2)


@pytest.mark.parametrize("nested", [False, True])
def test_quant_state_dict_round_trip(nested):
    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.utils import unpack_tensor_to_dict

    qs = _state(nested)
    packed = qs.as_dict(packed=True)
    key = "quant_state.bitsandbytes__nf4"
    assert key in packed and packed[key].dtype == torch.uint8
    assert all(isinstance(v, torch.Tensor) for v in packed.values())  # safetensors-ready
    meta = unpack_tensor_to_dict(packed[key])
    assert meta["quant_type"] == "nf4" and meta["blocksize"] == 64 and meta["shape"] == [64, 64]
    assert meta["dtype"] == ("float16" if nested else "bfloat16")
    if nested:
        assert set(packed) == {"absmax", "quant_map", "nested_absmax", "nested_quant_map", key}
        assert meta["nested_blocksize"] == 256 and abs(meta["nested_offset"] - 0.25) < 1e-7
    back = F.QuantState.from_dict({f"weight.{k}": v for k, v in packed.items()}, device="cpu")
    assert back == qs and back.nested == nested
    # FSDP-style getattr access to the packed key
    assert torch.equal(getattr(qs, "bitsandbytes__nf4"), packed[key])
    # legacy list view
    assert qs[3] == 64 and qs[5] == "nf4" and (qs[4] is None) == (not nested)
    with pytest.raises(ValueError):
        F.QuantState.from_dict({"absmax": qs.absmax}, device="cpu")


def test_pack_dict_is_plain_json():
    from bitsandbytes_b200.utils import pack_dict_to_tensor, unpack_tensor_to_dict

    d = {"quant_type": "fp4", "blocksize": 128, "shape": [3, 5], "nested_offset": 0.125}
    t = pack_dict_to_tensor(d)
    assert bytes(t.tolist()).decode() == '{"quant_type": "fp4", "blocksize": 128, "shape": [3, 5], "nested_offset": 0.125}'
    assert unpack_tensor_to_dict(t) == d


# ------------------------------------------------------------------------------------ schemas / shape functions
def test_every_reference_op_is_defined_with_the_reference_schema():
    import bitsandbytes_b200._ops as ops  # noqa: F401

    want = {
        "gemm_4bit": "bitsandbytes::gemm_4bit(Tensor A, Tensor B, int[] shapeB, Tensor absmax, int blocksize, str quant_type, "
                     "Tensor? bias=None, Tensor? absmax_8bit=None, Tensor? absmax_code=None, Tensor? absmax_offset=None) -> Tensor",
        "quantize_4bit": "bitsandbytes::quantize_4bit(Tensor A, int blocksize, str quant_type, ScalarType quant_storage) -> (Tensor, Tensor)",
        "int8_vectorwise_quant": "bitsandbytes::int8_vectorwise_quant(Tensor A, float threshold=0.) -> (Tensor, Tensor, Tensor?)",
    }
    for name, schema in want.items():
        got = str(getattr(torch.ops.bitsandbytes, name).default._schema)
        assert got.replace(" ", "") == schema.replace(" ", ""), got
    for name in ops.SCHEMAS:
        base, _, ov = name.partition(".")
        assert hasattr(getattr(torch.ops.bitsandbytes, base), ov or "default")


def test_shape_functions_under_fake_tensors():
    from torch._subclasses.fake_tensor import FakeTensorMode

    import bitsandbytes_b200._ops  # noqa: F401

    with FakeTensorMode():
        A = torch.empty(3, 7, 128, dtype=torch.bfloat16, device="cuda")
        B = torch.empty(64 * 128 // 2, 1, dtype=torch.uint8, device="cuda")
        absmax = torch.empty(64 * 128 // 64, dtype=torch.float32, device="cuda")
        y = torch.ops.bitsandbytes.gemm_4bit.default(A, B, [64, 128], absmax, 64, "nf4")
        assert y.shape == (3, 7, 64) and y.dtype == torch.bfloat16
        q, am = torch.ops.bitsandbytes.quantize_4bit.default(torch.empty(33, 65, device="cuda"), 64, "fp4", torch.bfloat16)
        assert q.shape == ((33 * 65 + 1) // 4, 1) and q.dtype == torch.bfloat16 and am.shape == (-(33 * 65 // -64),)
        q8, a8 = torch.ops.bitsandbytes.quantize_blockwise.default(torch.empty(1000, device="cuda"),
                                                                   torch.empty(256, device="cuda"), 256)
        assert q8.shape == (1000,) and q8.dtype == torch.uint8 and a8.shape == (4,)
        d = torch.ops.bitsandbytes.dequantize_4bit.default(B, absmax, 64, "nf4", [64, 128], torch.float16)
        assert d.shape == (64, 128) and d.dtype == torch.float16
        c = torch.ops.bitsandbytes.int8_linear_matmul.default(torch.empty(5, 32, dtype=torch.int8, device="cuda"),
                                                              torch.empty(9, 32, dtype=torch.int8, device="cuda"))
        assert c.shape == (5, 9) and c.dtype == torch.int32
        o = torch.ops.bitsandbytes.int8_mm_dequant.default(c, torch.empty(5, device="cuda"), torch.empty(9, device="cuda"))
        assert o.dtype == torch.float16
        with pytest.raises(Exception):
            torch.ops.bitsandbytes.gemm_4bit.default(A, B, [64, 128], absmax, 64, "int4")


# ------------------------------------------------------------------------------------ modules (host logic)
def _prequantized_linear(nested=False):
    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    qs = _state(nested)
    packed = torch.randint(0, 256, (64 * 64 // 2, 1), dtype=torch.uint8)
    m = bnb.nn.Linear4bit(64, 64, bias=True, quant_type="nf4", compress_statistics=nested)
    m.weight = bnb.nn.Params4bit.from_prequantized(packed, qs.as_dict(packed=True), device="cpu", module=m)
    return m, packed, qs


@pytest.mark.parametrize("nested", [False, True])
def test_linear4bit_state_dict_keys_and_reload(nested):
    import bitsandbytes_b200 as bnb

    m, packed, qs = _prequantized_linear(nested)
    sd = m.state_dict()
    expect = {"weight", "bias", "weight.absmax", "weight.quant_map", "weight.quant_state.bitsandbytes__nf4"}
    if nested:
        expect |= {"weight.nested_absmax", "weight.nested_quant_map"}
    assert set(sd) == expect
    stats = {k[len("weight."):]: v for k, v in sd.items() if k.startswith("weight.")}
    p2 = bnb.nn.Params4bit.from_prequantized(sd["weight"], stats, device="cpu")
    assert p2.quant_state == qs and torch.equal(p2.data, packed) and p2.bnb_quantized
    assert p2.blocksize == 64 and p2.quant_type == "nf4" and p2.compress_statistics == nested
    # FSDP-style attribute traversal
    assert torch.equal(m.weight.absmax, qs.absmax) and torch.equal(m.weight.quant_map, qs.code)
    if nested:
        assert torch.equal(m.weight.nested_absmax, qs.state2.absmax) and m.weight.nested_blocksize == 256
    else:
        with pytest.raises(AttributeError):
            m.weight.nested_absmax


def test_params4bit_copy_pickle_chunk():
    import copy

    m, packed, qs = _prequantized_linear()
    w = m.weight
    for clone in (copy.copy(w), copy.deepcopy(w)):
        assert type(clone).__name__ == "Params4bit"
    # pickling goes through Parameter.__reduce_ex__ (rebuilds a Parameter carrying our __dict__),
    # exactly as in the reference: the attributes survive (reference tests/test_linear4bit.py:316-345)
    for clone in (copy.copy(w), copy.deepcopy(w), pickle.loads(pickle.dumps(w))):
        assert torch.equal(clone.data, w.data) and not clone.requires_grad
        assert clone.quant_state == w.quant_state and clone.quant_type == "nf4" and clone.bnb_quantized
        assert set(clone.__dict__) == set(w.__dict__)
    assert copy.deepcopy(w).quant_state is not w.quant_state and copy.copy(w).quant_state is w.quant_state
    chunks = torch.chunk(w, 4, dim=0)
    assert all(type(c).__name__ == "Params4bit" and c.quant_state is w.quant_state for c in chunks)
    assert torch.equal(torch.cat([c.data for c in chunks]), w.data)  # shard round trip is lossless
    parts = torch.split(w, 512, dim=0)
    assert all(type(c).__name__ == "Params4bit" for c in parts)


def test_quant_storage_shard_round_trip():
    """reference tests/test_linear4bit.py:256-283: packed bytes viewed as quant_storage, flattened,
    chunked (FSDP) and reassembled are the same bytes."""
    packed = torch.randint(0, 256, (4096,), dtype=torch.uint8)
    for dt in (torch.bfloat16, torch.float16, torch.float32):
        stored = packed.view(dt)
        shards = torch.chunk(stored.flatten(), 4)
        assert torch.equal(torch.cat(shards).view(torch.uint8), packed)


def test_fix_quant_state_from_module():
    import bitsandbytes_b200 as bnb

    m, packed, qs = _prequantized_linear()
    m.weight = torch.nn.Parameter(m.weight.data.clone(), requires_grad=False)  # what FSDP does
    assert getattr(m.weight, "quant_state", None) is None
    bnb.nn.fix_4bit_weight_quant_state_from_module(m)
    assert isinstance(m.weight, bnb.nn.Params4bit) and m.weight.quant_state is m.quant_state


def test_linear8bitlt_state_dict_and_format_hook():
    import bitsandbytes_b200 as bnb

    m = bnb.nn.Linear8bitLt(32, 16, bias=False, has_fp16_weights=False, threshold=6.0)
    assert m.state.threshold == 6.0 and m.state.use_pool and not m.weight.requires_grad
    CB = torch.randint(-127, 128, (16, 32), dtype=torch.int8)
    SCB = torch.rand(16) + 0.5
    m.weight = bnb.nn.Int8Params(CB, requires_grad=False, has_fp16_weights=False, CB=CB, SCB=SCB)
    sd = m.state_dict()
    assert set(sd) == {"weight", "SCB", "weight_format"} and sd["weight_format"].item() == 0
    m2 = bnb.nn.Linear8bitLt(32, 16, bias=False, has_fp16_weights=False)
    m2.weight = bnb.nn.Int8Params(torch.zeros(16, 32, dtype=torch.int8), requires_grad=False, CB=None,
                                  SCB=torch.zeros(16))
    m2.load_state_dict(sd)
    assert torch.equal(m2.weight.data, CB) and torch.equal(m2.weight.SCB, SCB)
    bad = dict(sd)
    bad["weight_format"] = torch.tensor(2, dtype=torch.uint8)
    with pytest.raises(ValueError):
        m2.load_state_dict(bad)
    m3 = bnb.nn.Linear8bitLt(32, 16, bias=False, has_fp16_weights=False)
    with pytest.raises(RuntimeError):
        m3.load_state_dict(sd)  # not quantised yet: no SCB buffer to load into


def test_matmul_4bit_argument_errors():
    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    with pytest.raises(ValueError):
        bnb.matmul_4bit(torch.randn(2, 64), torch.zeros(2048, 1, dtype=torch.uint8), None)
    qs = F.QuantState(absmax=torch.rand(64), shape=torch.Size([4096]), code=None, blocksize=64, quant_type="nf4")
    with pytest.raises(ValueError):
        bnb.matmul_4bit(torch.randn(2, 64), torch.zeros(2048, 1, dtype=torch.uint8), qs)
    # empty input: no kernel needed
    qs2 = _state(False)
    out = bnb.matmul_4bit(torch.empty(0, 64), torch.zeros(2048, 1, dtype=torch.uint8), qs2)
    assert out.shape == (0, 64)


# ------------------------------------------------------------------------------------ sharding (N > 1 path)
def _global_problem():
    import oracle

    g = torch.Generator().manual_seed(7)
    N, K, M = 1024, 128, 6
    W = (torch.randn(N, K, generator=g) / K**0.5).to(torch.bfloat16)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16)
    packed, absmax = oracle.quantize_blockwise(W.float().numpy().reshape(-1), 64, "fp4")
    return N, K, M, x, torch.from_numpy(packed), torch.from_numpy(absmax)


def _nested_state(absmax, N, K):
    import bitsandbytes_b200.functional as F
    import oracle

    offset = absmax.mean()
    code2 = F.create_dynamic_map()
    a8, a2 = oracle.quantize_blockwise((absmax - offset).numpy(), 256, None, code2.numpy())
    s2 = F.QuantState(absmax=torch.from_numpy(a2), code=code2, blocksize=256, dtype=torch.float32)
    return F.QuantState(absmax=torch.from_numpy(a8), shape=torch.Size([N, K]), code=F.get_4bit_type("fp4", "cpu"),
                        blocksize=64, quant_type="fp4", dtype=torch.bfloat16, offset=offset, state2=s2)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("nested", [False, True])
def test_row_slices_reproduce_the_global_weight(world, nested):
    """Slicing a globally quantised weight by rows is lossless: dequantising the shards with the
    oracle and stacking them gives the dequantised global weight, bit for bit (incl. double quant)."""
    import bitsandbytes_b200.functional as F
    import oracle
    from bitsandbytes_b200.parallel import reassemble_shards, slice_quantized_weight

    N, K, M, x, packed, absmax = _global_problem()
    if nested:
        qs = _nested_state(absmax, N, K)
        scale = oracle.nested_absmax(qs.state2.absmax.numpy(), qs.absmax.numpy(), qs.state2.code.numpy(), float(qs.offset))
    else:
        qs = F.QuantState(absmax=absmax, shape=torch.Size([N, K]), code=None, blocksize=64, quant_type="fp4",
                          dtype=torch.bfloat16)
        scale = absmax.numpy()
    full = oracle.dequantize_blockwise(packed.numpy(), scale, 64, N * K, "fp4", None, "bf16").reshape(N, K)
    rows = []
    shards = [slice_quantized_weight(packed, qs, world, r) for r in range(world)]
    for s in shards:
        if nested:
            sc = oracle.nested_absmax(s.absmax.numpy(), s.absmax_8bit.numpy(), s.absmax_code.numpy(),
                                      float(s.absmax_offset))
        else:
            sc = s.absmax.numpy()
        rows.append(oracle.dequantize_blockwise(s.packed.numpy(), sc, 64, s.rows * K, "fp4", None, "bf16").reshape(s.rows, K))
    assert np.array_equal(np.concatenate(rows), full)
    if not nested:
        p, a = reassemble_shards(shards)
        assert torch.equal(p, packed) and torch.equal(a, absmax)


def test_shard_alignment_errors():
    import bitsandbytes_b200.functional as F
    from bitsandbytes_b200.parallel import slice_quantized_weight

    N, K, M, x, packed, absmax = _global_problem()
    qs = F.QuantState(absmax=absmax, shape=torch.Size([N, K]), code=None, blocksize=64, quant_type="fp4")
    with pytest.raises(ValueError):
        slice_quantized_weight(packed, qs, 3, 0)          # 1024 % 3
    with pytest.raises(ValueError):
        slice_quantized_weight(packed, _nested_state(absmax, N, K), 16, 0)  # 64 rows * 2 blocks = 128 < 256


WORKER = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["REPO_ROOT"])
import oracle
import bitsandbytes_b200.functional as F
from bitsandbytes_b200 import parallel
from tests.test_host_cpu import _global_problem

def oracle_local_forward(self, x, out=None, ldc=None):
    # test-only stand-in for the CUDA kernel: the CPU oracle computes this rank's slice
    s = self.shard
    M = x.numel() // s.K
    y = oracle.gemm_4bit(x.float().numpy().reshape(-1), s.packed.numpy(), s.absmax.numpy(), M, s.rows, s.K,
                         s.blocksize, s.quant_type, "bf16")
    y = torch.from_numpy(y).to(torch.bfloat16)
    if out is None:
        return y
    out.copy_(y)
    return out

dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % os.environ["PORT"],
                        rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
N, K, M, x, packed, absmax = _global_problem()
qs = F.QuantState(absmax=absmax, shape=torch.Size([N, K]), code=None, blocksize=64, quant_type="fp4", dtype=torch.bfloat16)
parallel.ColumnParallelLinear4bit.local_forward = oracle_local_forward
layer = parallel.ColumnParallelLinear4bit.from_quantized(packed, qs)
y = layer(x)
full = torch.from_numpy(oracle.gemm_4bit(x.float().numpy().reshape(-1), packed.numpy(), absmax.numpy(), M, N, K, 64,
                                         "fp4", "bf16")).to(torch.bfloat16)
assert y.shape == (M, N), y.shape
assert torch.equal(y, full), (y - full).abs().max()
local = parallel.ColumnParallelLinear4bit.from_quantized(packed, qs, gather_output=False)(x)
r, w = dist.get_rank(), dist.get_world_size()
assert torch.equal(local, full[:, r * N // w:(r + 1) * N // w])
dist.barrier()
dist.destroy_process_group()
print("OK", r)
'''


def test_column_parallel_linear_world_size_2_gloo(tmp_path):
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", PORT=str(port), REPO_ROOT=str(ROOT), OMP_NUM_THREADS="2")
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True, cwd=ROOT))
    outs = [p.communicate(timeout=240)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"OK {r}" in o, o[-3000:]


# ----------------------------------------------------------------------------------------------
# Checkpoints written by the REFERENCE load into our modules and serialise back to the same bytes
# (fixtures: tests/golden/make_golden_state_dicts.py, generated by importing the reference here)
# ----------------------------------------------------------------------------------------------
_TORCH_DT = {"torch.float32": torch.float32, "torch.bfloat16": torch.bfloat16, "torch.float16": torch.float16,
             "torch.uint8": torch.uint8, "torch.int8": torch.int8, "torch.int64": torch.int64}


def _reference_state_dict(case):
    z = np.load(ROOT / "tests" / "golden" / "reference_state_dicts.npz")
    sd, extra = {}, {}
    for k in z.files:
        if not k.startswith(case + "::"):
            continue
        name = k.split("::", 1)[1]
        if name.startswith("__dtype__"):
            continue
        if name.startswith("__"):
            extra[name] = z[k]
            continue
        dt = _TORCH_DT[str(z[f"{case}::__dtype__{name}"])]
        arr = z[k]
        t = torch.from_numpy(arr.view(np.int16).copy()).view(dt) if dt in (torch.bfloat16, torch.float16) else \
            torch.from_numpy(arr.copy())
        assert t.dtype == dt, (name, t.dtype, dt)
        sd[name] = t
    return sd, extra


@pytest.mark.parametrize("case,qt,nested,storage", [
    ("l4_nf4_plain", "nf4", False, torch.uint8), ("l4_nf4_nested", "nf4", True, torch.uint8),
    ("l4_fp4_plain", "fp4", False, torch.uint8), ("l4_nf4_bf16storage", "nf4", False, torch.bfloat16)])
def test_reference_linear4bit_checkpoint_round_trips(case, qt, nested, storage):
    import bitsandbytes_b200 as bnb

    ref_sd, extra = _reference_state_dict(case)
    bs, is_nested, K, N = (int(v) for v in extra["__meta__"])
    assert bool(is_nested) == nested
    m = bnb.nn.Linear4bit(K, N, bias=True, compute_dtype=torch.bfloat16, compress_statistics=nested, quant_type=qt,
                          quant_storage=storage)
    # the route HF Transformers takes for a pre-quantised checkpoint (and reference tests/test_linear4bit.py:60-75):
    # Params4bit.from_prequantized(data, quantized_stats) -- the reference's Linear4bit has no load hook either
    stats = {k[len("weight."):]: v for k, v in ref_sd.items() if k.startswith("weight.")}
    m.weight = bnb.nn.Params4bit.from_prequantized(data=ref_sd["weight"], quantized_stats=stats, device="cpu",
                                                   module=m)
    with torch.no_grad():
        m.bias.copy_(ref_sd["bias"])
    w = m.weight
    assert w.bnb_quantized and w.quant_state is not None
    qs = w.quant_state
    assert (qs.blocksize, qs.quant_type, tuple(qs.shape), qs.nested) == (bs, qt, (N, K), nested)
    assert qs.dtype == torch.float32  # the layer was quantised from an fp32 nn.Linear
    assert w.dtype == storage and w.numel() * w.element_size() == N * K // 2
    out_sd = m.state_dict()
    assert set(out_sd) == set(ref_sd)
    for k, v in ref_sd.items():
        got = out_sd[k]
        assert got.dtype == v.dtype and got.shape == v.shape, k
        assert torch.equal(got.view(torch.uint8) if got.dtype != torch.uint8 else got,
                           v.view(torch.uint8) if v.dtype != torch.uint8 else v), k


def test_reference_linear8bitlt_checkpoint_round_trips():
    import bitsandbytes_b200 as bnb

    ref_sd, extra = _reference_state_dict("l8")
    N, K = extra["__float_weight__"].shape
    m = bnb.nn.Linear8bitLt(K, N, bias=True, has_fp16_weights=False, threshold=6.0)
    with pytest.raises(RuntimeError, match="non-quantized Linear8bitLt"):  # the reference's rule (nn/modules.py:1111-1116)
        m.load_state_dict(ref_sd, strict=True)
    # a quantised (int8 + SCB) module accepts the checkpoint: on a GPU `.cuda()` puts it in that state, here the
    # int8 parameter is installed directly, the way Transformers' bnb quantizer does for pre-quantised weights
    m.weight = bnb.nn.Int8Params(torch.zeros(N, K, dtype=torch.int8), requires_grad=False, has_fp16_weights=False,
                                 SCB=torch.zeros(N))
    missing, unexpected = m.load_state_dict(ref_sd, strict=True)
    assert not missing and not unexpected
    assert m.weight.dtype == torch.int8 and torch.equal(m.weight.data, ref_sd["weight"])
    assert m.weight.SCB is not None and torch.equal(m.weight.SCB, ref_sd["SCB"])
    # the row statistics are the row absmax of the fp16-cast weight (reference Int8Params._quantize casts first)
    W = torch.from_numpy(extra["__float_weight__"]).half()
    assert torch.equal(W.abs().amax(dim=1).float(), ref_sd["SCB"])
    out_sd = m.state_dict()
    assert set(out_sd) == set(ref_sd)
    for k, v in ref_sd.items():
        assert out_sd[k].dtype == v.dtype and torch.equal(out_sd[k], v), k


def _codebook_cases():
    sys.path.insert(0, str(ROOT / "tests" / "golden"))
    try:
        import make_golden_codebooks as g
    finally:
        sys.path.pop(0)
    return g


def test_code_book_builders_match_the_reference_bit_for_bit():
    """create_linear_map / create_fp8_map / create_dynamic_map / create_normal_map against goldens generated by the
    reference for a spread of parameters (tests/golden/make_golden_codebooks.py)."""
    import bitsandbytes_b200.functional as F

    g = _codebook_cases()
    z = np.load(ROOT / "tests" / "golden" / "reference_codebooks.npz")

    def same(name, ours):
        ref = z[name]
        got = ours.numpy()
        assert got.dtype == ref.dtype and got.shape == ref.shape, name
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (name, np.abs(got - ref).max())

    for a in g.LINEAR:
        same("linear_" + "_".join(str(int(v)) for v in a), F.create_linear_map(*a))
    for a in g.FP8:
        same("fp8_" + "_".join(str(int(v)) for v in a), F.create_fp8_map(*a))
    for a in g.DYNAMIC:
        same("dynamic_" + "_".join(str(int(v)) for v in a), F.create_dynamic_map(*a))
    for off, extra in g.NORMAL:
        same(f"normal_{off}_{int(extra)}", F.create_normal_map(off, extra))


def test_fused_forward_rejects_a_mismatched_gather_buffer_before_any_launch():
    """parallel.fused_forward validates the symmetric-memory slot against the layer on the host."""
    from types import SimpleNamespace

    from bitsandbytes_b200 import parallel

    shard = parallel.Shard4bit(packed=torch.zeros(8 * 64 // 2, dtype=torch.uint8), absmax=torch.zeros(8), absmax_8bit=None,
                               absmax_code=None, absmax_offset=None, rows=8, row0=0, K=64, blocksize=64, quant_type="nf4")
    layer = parallel.ColumnParallelLinear4bit(shard, out_features=16)
    x = torch.zeros(4, 64, dtype=torch.bfloat16)
    for peers in (SimpleNamespace(M=5, N=16, dtype=torch.bfloat16), SimpleNamespace(M=4, N=32, dtype=torch.bfloat16),
                  SimpleNamespace(M=4, N=16, dtype=torch.float16)):
        with pytest.raises(ValueError, match="different output shape"):
            parallel.fused_forward(layer, x, peers)


def test_transformers_swaps_in_our_modules_through_the_import_shim():
    """shim/ on PYTHONPATH: Hugging Face Transformers' bitsandbytes integration (replace_with_bnb_linear,
    BitsAndBytesConfig) sees `bitsandbytes` >= 0.46.1 and builds OUR Linear4bit / Linear8bitLt modules --
    host logic only (meta device), so it runs without a GPU."""
    pytest.importorskip("transformers")
    code = r'''
import json, torch
from transformers.utils import is_bitsandbytes_available
assert is_bitsandbytes_available()
import bitsandbytes, bitsandbytes_b200
assert bitsandbytes is bitsandbytes_b200
from transformers import LlamaConfig, LlamaForCausalLM, BitsAndBytesConfig
from transformers.integrations.bitsandbytes import replace_with_bnb_linear
cfg = LlamaConfig(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                  num_key_value_heads=2, vocab_size=512)
out = {}
for tag, qc in (("4bit", BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type="nf4",
                                             bnb_4bit_compute_dtype=torch.bfloat16, bnb_4bit_use_double_quant=True)),
                ("8bit", BitsAndBytesConfig(load_in_8bit=True, llm_int8_threshold=6.0))):
    with torch.device("meta"):
        model = LlamaForCausalLM(cfg)
    model = replace_with_bnb_linear(model, modules_to_not_convert=["lm_head"], quantization_config=qc)
    mods = [(n, type(m).__module__, type(m).__name__) for n, m in model.named_modules()
            if type(m).__name__ in ("Linear4bit", "Linear8bitLt", "Linear")]
    q = model.model.layers[0].self_attn.q_proj
    out[tag] = {"mods": mods, "weight": type(q.weight).__name__,
                "detail": [q.weight.quant_type, q.weight.compress_statistics, str(q.compute_dtype)] if tag == "4bit"
                else [float(q.state.threshold), bool(q.state.has_fp16_weights)]}
print(json.dumps(out))
'''
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(ROOT / "shim"), str(ROOT), os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600, cwd="/tmp")
    assert r.returncode == 0, r.stderr[-3000:]
    import json

    out = json.loads(r.stdout.strip().splitlines()[-1])
    for tag, cls, wcls in (("4bit", "Linear4bit", "Params4bit"), ("8bit", "Linear8bitLt", "Int8Params")):
        mods = out[tag]["mods"]
        ours = [m for m in mods if m[2] == cls]
        assert len(ours) == 14 and all(m[1].startswith("bitsandbytes_b200.") for m in ours)
        assert [m[0] for m in mods if m[2] == "Linear"] == ["lm_head"]
        assert out[tag]["weight"] == wcls
    assert out["4bit"]["detail"] == ["nf4", True, "torch.bfloat16"]
    assert out["8bit"]["detail"] == [6.0, False]
