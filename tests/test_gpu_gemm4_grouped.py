"""GPU: the grouped 4-bit GEMM (every expert of a mixture-of-experts layer in one launch) through the C ABI, the op,
bnb.grouped_matmul_4bit and bnb.nn.GroupedLinear4bit.

Each expert's rows must equal, bit for bit, the plain wgmma kernel on that expert alone at the same token tile with no
K split (cbnb_b200_gemm_4bit_pair on A[s:e] against the flattened weight, whose columns [e*N, (e+1)*N) are the
expert's), and every row must be within the suite's bound of the float64 oracle (test_gpu_gemm4.assert_close_to_exact).
Outputs start NaN-filled, with guard elements past their end that must stay untouched; rows past offs[E-1] must read
back as zeros.
"""
import ctypes as ct
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import _native as nat
from tests.test_gpu_gemm4 import assert_close_to_exact, exact, make_problem

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
GUARD = 64
MTS = [16, 32, 64, 128]


def grouped_mt(p, E, offs, mt, ldc=None, shift=0, entry="mt"):
    """The grouped entry on make_problem's [E*N, K] problem; returns (out [M, N] view, the whole NaN-filled buffer).
    shift: elements by which the output base is moved off its 16-byte alignment (the element-wise store path)."""
    M, N, K = p["M"], p["N"] // E, p["K"]
    ldc = ldc or N
    buf = torch.full((shift + M * ldc + GUARD,), float("nan"), dtype=nat.DTYPE[p["dtype"]], device="cuda")
    out = buf[shift:shift + M * ldc].view(M, ldc)[:, :N]
    offs_t = offs if isinstance(offs, torch.Tensor) else torch.tensor(offs, dtype=torch.int32, device="cuda")
    args = [nat.ptr(p["x"]), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]),
            nat.ptr(p["absmax_code"]), nat.ptr(p["absmax_offset"]), offs_t.data_ptr(), E, out.data_ptr(),
            nat.ptr(p["bias"]), M, N, K, ldc, p["bs"], nat.QT_ID[p["qt"]], nat.DTYPE_ID[p["dtype"]]]
    if entry == "mt":
        rc = nat.lib.cbnb_b200_gemm_4bit_grouped_mt(*args, mt, nat.stream())
    else:
        rc = nat.lib.cbnb_b200_gemm_4bit_grouped(*args, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0, rc
    return out, buf


def pair(p, s, e, mt):
    """The plain kernel on rows [s, e) against the whole flattened weight, token tile mt, no K split."""
    NE, K = p["N"], p["K"]
    out = torch.full((e - s, NE), float("nan"), dtype=nat.DTYPE[p["dtype"]], device="cuda")
    x = p["x"][s:e]
    rc = nat.lib.cbnb_b200_gemm_4bit_pair(
        x.data_ptr(), nat.ptr(p["packed"]), nat.ptr(p["absmax"]), nat.ptr(p["absmax_8bit"]), nat.ptr(p["absmax_code"]),
        nat.ptr(p["absmax_offset"]), out.data_ptr(), nat.ptr(p["bias"]), e - s, NE, K, NE, p["bs"],
        nat.QT_ID[p["qt"]], nat.DTYPE_ID[p["dtype"]], mt, 1, None, nat.stream())
    torch.cuda.synchronize()
    nat.check()
    assert rc == 0, rc
    return out


def clamp_ends(offs, M):
    ends, run = [], 0
    for o in offs:
        run = min(max(o, run), M)
        ends.append(run)
    return ends


def check_grouped(p, E, offs, mt, got, buf, oracle=True, shift=0):
    """Bit for bit against the per-expert plain kernel, within the bound of the oracle, zeros past the last end, guard
    elements untouched."""
    M, N = p["M"], p["N"] // E
    ends = clamp_ends(offs, M)
    start = 0
    for e, end in enumerate(ends):
        if end > start:
            want = pair(p, start, end, mt)[:, e * N:(e + 1) * N]
            assert torch.equal(got[start:end], want), f"expert {e} rows [{start}, {end}) differ from the plain kernel"
        start = end
    assert (got[ends[-1]:] == 0).all(), "rows past the last expert's end are not zero"
    assert torch.isnan(buf[buf.numel() - GUARD:]).all() and torch.isnan(buf[:shift]).all(), "guard elements written"
    if oracle and ends[-1] > 0:
        y64 = exact(dict(p, M=ends[-1], x=p["x"][:ends[-1]]))
        want = np.concatenate([y64[s:t, e * N:(e + 1) * N] for e, (s, t) in enumerate(zip([0] + ends[:-1], ends))])
        assert_close_to_exact(got[:ends[-1]], want, p["dtype"], p["K"])


def routing(counts, tail=0):
    ends = np.cumsum(counts).tolist()
    return ends, ends[-1] + tail


# ---------------------------------------------------------------------------------------------------- every instance
@pytest.mark.parametrize("mt", MTS)
@pytest.mark.parametrize("nested", [False, True], ids=["plain", "nested"])
@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
def test_every_instance(dtype, qt, nested, mt, bias):
    """Counts of MT + 3, 0 (an empty expert in the middle), 1 and 2 MT - 1 (below / not a multiple of MT), 5 tail rows;
    N = 192, so that the second n-tile of an expert reaches into the next expert's codes."""
    E, N, K = 4, 192, 512
    offs, M = routing([mt + 3, 0, 1, 2 * mt - 1], tail=5)
    p = make_problem(M, E * N, K, qt, dtype, bs=64, nested=nested, bias=bias, seed=mt)
    got, buf = grouped_mt(p, E, offs, mt)
    check_grouped(p, E, offs, mt, got, buf)


# ---------------------------------------------------------------------------------------------------- routings
ROUTINGS = {
    "uniform": dict(E=8, N=256, K=256, counts=[40] * 8, mt=32),
    "skewed": dict(E=8, N=256, K=256, counts=[0, 0, 0, 300, 0, 0, 0, 0], mt=64),
    "empty_first": dict(E=6, N=128, K=256, counts=[0, 0, 17, 33, 64, 1], mt=32),
    "empty_last": dict(E=6, N=128, K=256, counts=[17, 33, 64, 1, 0, 0], mt=16),
    "single_rows": dict(E=16, N=128, K=128, counts=[1] * 16, mt=16, tail=3),
    "one_expert": dict(E=1, N=384, K=512, counts=[77], mt=64),
    "n200": dict(E=5, N=200, K=256, counts=[30, 9, 0, 70, 2], mt=32, tail=7),
    "blocks_mid_row": dict(E=4, N=200, K=576, counts=[20, 50, 3, 40], mt=32, bs=128),
    "experts_mid_block": dict(E=4, N=200, K=576, counts=[20, 50, 3, 40], mt=64, bs=4096),
    "more_units_than_sms": dict(E=8, N=2048, K=256, counts=[128] * 8, mt=16),
    "m128": dict(E=3, N=256, K=1024, counts=[300, 129, 128], mt=128, tail=1),
}


@pytest.mark.parametrize("name", list(ROUTINGS))
def test_routings(name):
    r = ROUTINGS[name]
    E, N, K, mt = r["E"], r["N"], r["K"], r["mt"]
    offs, M = routing(r["counts"], r.get("tail", 0))
    p = make_problem(M, E * N, K, "nf4", "bf16", bs=r.get("bs", 64), bias=True, seed=len(name))
    got, buf = grouped_mt(p, E, offs, mt)
    check_grouped(p, E, offs, mt, got, buf)
    if E == 1:  # one expert: the plain kernel on all its rows at the same tile
        assert torch.equal(got[:offs[0]], pair(p, 0, offs[0], mt))


@pytest.mark.parametrize("ldc,shift", [(200, 0), (203, 0), (192, 1)])
def test_strided_and_misaligned_output(ldc, shift):
    """ldc > N, and an output base off 16 bytes: the element-wise store path, same bits."""
    E, N, K = 4, 192, 256
    offs, M = routing([33, 0, 70, 5], tail=4)
    p = make_problem(M, E * N, K, "fp4", "fp16", bias=True, seed=7)
    got, buf = grouped_mt(p, E, offs, 32, ldc=ldc, shift=shift)
    check_grouped(p, E, offs, 32, got, buf, shift=shift)
    # the columns between N and ldc are never written
    if ldc > N:
        pad = buf[shift:shift + M * ldc].view(M, ldc)[:, N:]
        assert torch.isnan(pad).all()


@pytest.mark.parametrize("offs", [[40, 20, 90, 60], [-5, 30, -1, 70], [30, 200, 10, 500], [-3, -3, -3, -3]],
                         ids=["decreasing", "negative", "past_m", "all_negative"])
def test_malformed_offs_are_clamped(offs):
    E, N, K, M = 4, 192, 256, 100
    p = make_problem(M, E * N, K, "nf4", "bf16", bias=True, seed=9)
    got, buf = grouped_mt(p, E, offs, 32)
    want, _ = grouped_mt(p, E, clamp_ends(offs, M), 32)
    assert torch.equal(got, want)
    check_grouped(p, E, offs, 32, got, buf)


# ---------------------------------------------------------------------------------------------------- production entry
def rule_tile(M, E):
    want = 2 * -(M // -E)  # twice the mean rows per expert
    return 16 if want <= 16 else 32 if want <= 32 else 64 if want <= 64 else 128


PROD_CASES = [(1, 8), (64, 8), (200, 8), (512, 8), (1024, 8), (4096, 16)]


def record_tiles_main():
    """The child: runs the production op for each (M, E) of PROD_CASES under torch.profiler and prints the token tile
    of every grouped kernel instance it launched (the profiler stays out of the pytest process)."""
    import re

    from torch.profiler import ProfilerActivity, profile

    import bitsandbytes_b200  # noqa: F401
    import bitsandbytes_b200.functional as F

    res = {}
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device="cuda").add_(1)
            torch.cuda.synchronize()
    for M, E in PROD_CASES:
        N, K = 256, 256
        W = torch.randn(E, N, K, device="cuda", dtype=torch.bfloat16)
        qW, qs = F.quantize_4bit(W, quant_type="nf4")
        x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        offs = torch.tensor(np.linspace(0, M, E + 1)[1:].round(), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.ops.bitsandbytes.gemm_4bit_grouped(x, qW, qs.shape, qs.absmax, qs.blocksize, "nf4", offs)
            torch.cuda.synchronize()
        tiles = []
        for ev in prof.events():
            m = re.search(r"gemm4_tc_kernel<([^<>]*)>", ev.name)
            if m and ev.device_type == torch.autograd.DeviceType.CUDA:
                args = [re.sub(r"^\((?:bool|int)\)", "", a.strip()) for a in m.group(1).split(",")]
                tiles.append([args[2], args[-1]])
        res[f"{M},{E}"] = tiles
    print("TILES " + json.dumps(res), flush=True)


def test_production_entry_takes_the_rule_tile():
    """The production output equals the _mt entry at the rule's tile, bit for bit; and the tile the rule picks is proven
    from the kernel name."""
    for M, E in PROD_CASES:
        offs, _ = routing(np.diff(np.linspace(0, M, E + 1).round()).astype(int).tolist())
        p = make_problem(M, E * 256, 256, "nf4", "bf16", bias=True, seed=M)
        a, _ = grouped_mt(p, E, offs, 0, entry="prod")
        b, _ = grouped_mt(p, E, offs, rule_tile(M, E))
        assert torch.equal(a, b)
    code = (f"import sys; sys.path.insert(0, {str(ROOT)!r}); "
            "from tests.test_gpu_gemm4_grouped import record_tiles_main; record_tiles_main()")
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code],
                       capture_output=True, text=True, timeout=600)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("TILES ")]
    assert line, r.stdout[-2000:] + r.stderr[-2000:]
    tiles = json.loads(line[0][6:])
    for M, E in PROD_CASES:
        got = tiles[f"{M},{E}"]
        if not got:
            pytest.skip("torch.profiler recorded no CUDA kernels here: which kernel instance ran is not confirmed")
        assert got == [[str(rule_tile(M, E)), "1"]] or got == [[str(rule_tile(M, E)), "true"]], (M, E, got)


# ---------------------------------------------------------------------------------------------------- Python layers
def _expert_weight(E, N, K, dtype=torch.bfloat16, nested=False, qt="nf4", seed=0):
    import bitsandbytes_b200.functional as F

    g = torch.Generator(device="cuda").manual_seed(seed)
    W = (torch.randn(E, N, K, device="cuda", generator=g) / K**0.5).to(dtype)
    qW, qs = F.quantize_4bit(W, quant_type=qt, compress_statistics=nested)
    return qW, qs


def _op_reference(x, qW, qs, offs_list, bias):
    """The same call through the C entry at the rule tile (nat.lib), as a bit-for-bit reference for the Python layers."""
    import bitsandbytes_b200.functional as F

    Wd = F.dequantize_4bit(qW, qs)
    E, N, K = qs.shape
    M = x.shape[0]
    out = torch.zeros(M, N, dtype=x.dtype, device="cuda")
    ends = clamp_ends(offs_list, M)
    s = 0
    for e, t in enumerate(ends):
        if t > s:
            y = x[s:t].double() @ Wd[e].double().t()
            if bias is not None:
                y = y + bias[e].double()
            out[s:t] = y.to(x.dtype)
        s = t
    return out, ends


def test_op_and_autograd_forward_match_the_c_entry():
    import bitsandbytes_b200 as bnb

    E, N, K = 8, 256, 512
    qW, qs = _expert_weight(E, N, K, nested=True)
    offs_list, M = routing([10, 0, 40, 3, 70, 1, 0, 9], tail=6)
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    bias = torch.randn(E, N, device="cuda", dtype=torch.bfloat16)
    offs = torch.tensor(offs_list, dtype=torch.int32, device="cuda")
    y = bnb.grouped_matmul_4bit(x, qW, qs, offs, bias=bias)
    p = dict(x=x, packed=qW, absmax=qs.state2.absmax, absmax_8bit=qs.absmax, absmax_code=qs.state2.code,
             absmax_offset=qs.offset.reshape(1).float(), M=M, N=E * N, K=K, bs=qs.blocksize, qt="nf4", dtype="bf16",
             bias=bias.reshape(-1))
    want, _ = grouped_mt(p, E, offs_list, rule_tile(M, E))
    assert torch.equal(y, want)
    ref, ends = _op_reference(x, qW, qs, offs_list, bias)
    assert torch.allclose(y[:ends[-1]].float(), ref[:ends[-1]].float(), rtol=2e-2, atol=2e-2)
    assert (y[ends[-1]:] == 0).all()
    # M = 0: an empty [0, N] result without a launch
    assert bnb.grouped_matmul_4bit(x[:0], qW, qs, offs).shape == (0, N)


def test_cuda_graph_replays_new_routings_in_place():
    import bitsandbytes_b200 as bnb

    E, N, K, M = 8, 384, 256, 96
    qW, qs = _expert_weight(E, N, K, seed=1)
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    offs = torch.tensor(routing([12] * 8)[0], dtype=torch.int32, device="cuda")
    bnb.grouped_matmul_4bit(x, qW, qs, offs)  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            y = bnb.grouped_matmul_4bit(x, qW, qs, offs)
    torch.cuda.current_stream().wait_stream(s)
    for counts, tail in (([96, 0, 0, 0, 0, 0, 0, 0], 0), ([0, 5, 17, 0, 33, 1, 2, 30], 8), ([1] * 8, 88)):
        new = torch.tensor(routing(counts, tail)[0], dtype=torch.int32, device="cuda")
        offs.copy_(new)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, bnb.grouped_matmul_4bit(x, qW, qs, new))


@pytest.mark.parametrize("tail", [0, 5])
def test_autograd_bf16_against_float64(tail):
    import bitsandbytes_b200 as bnb
    import bitsandbytes_b200.functional as F

    E, N, K = 6, 256, 320
    qW, qs = _expert_weight(E, N, K, nested=False, seed=2)
    offs_list, M = routing([30, 0, 7, 64, 1, 19], tail=tail)
    offs = torch.tensor(offs_list, dtype=torch.int32, device="cuda")
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    bias = torch.randn(E, N, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    y = bnb.grouped_matmul_4bit(x, qW, qs, offs, bias=bias)
    go = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    y.backward(go)
    Wd = F.dequantize_4bit(qW, qs).double()
    gA = torch.zeros(M, K, dtype=torch.float64, device="cuda")
    gb = torch.zeros(E, N, dtype=torch.float64, device="cuda")
    s = 0
    for e, t in enumerate(offs_list):
        gA[s:t] = go[s:t].double() @ Wd[e]
        gb[e] = go[s:t].double().sum(0)
        s = t
    assert (x.grad[offs_list[-1]:] == 0).all()
    tol = 2.0**-7 * gA.abs() + 2.0**-12 * (N**0.5)
    assert ((x.grad.double() - gA).abs() <= tol).all()
    tolb = 2.0**-7 * gb.abs() + 2.0**-20 * M
    assert ((bias.grad.double() - gb).abs() <= tolb).all()


def test_fp16_training_is_refused():
    import bitsandbytes_b200 as bnb

    qW, qs = _expert_weight(2, 128, 128, dtype=torch.float16)
    x = torch.randn(4, 128, device="cuda", dtype=torch.float16, requires_grad=True)
    offs = torch.tensor([2, 4], dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="bfloat16"):
        bnb.grouped_matmul_4bit(x, qW, qs, offs)
    with torch.no_grad():
        assert bnb.grouped_matmul_4bit(x, qW, qs, offs).shape == (4, 128)


@pytest.mark.parametrize("nested", [False, True], ids=["plain", "nested"])
def test_grouped_linear4bit(nested):
    import bitsandbytes_b200 as bnb
    from bitsandbytes_b200.nn import GroupedLinear4bit, Linear4bit, Params4bit

    E, K, N = 4, 256, 192
    m = GroupedLinear4bit(E, K, N, bias=True, compress_statistics=nested, quant_type="nf4")
    W = m.weight.data.clone()
    m = m.cuda()
    assert m.weight.bnb_quantized and tuple(m.weight.quant_state.shape) == (E, N, K)
    assert m.weight.quant_state.nested == nested
    offs_list, M = routing([20, 0, 33, 9], tail=2)
    offs = torch.tensor(offs_list, dtype=torch.int32, device="cuda")
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        y = m(x, offs)
    assert y.dtype == torch.bfloat16 and y.shape == (M, N)
    assert torch.equal(y, bnb.grouped_matmul_4bit(x, m.weight, m.weight.quant_state, offs, bias=m.bias))
    ref, ends = _op_reference(x, m.weight, m.weight.quant_state, offs_list, m.bias)
    assert torch.allclose(y[:ends[-1]].float(), ref[:ends[-1]].float(), rtol=2e-2, atol=2e-2)
    # the quantised weight is the expert tensor's: dequantising it gives back W to 4-bit precision
    assert (W.cuda().float() - bnb.functional.dequantize_4bit(m.weight, m.weight.quant_state).float()).abs().max() < 0.1

    sd = m.state_dict()
    lin = Linear4bit(K, N, bias=True, compress_statistics=nested, quant_type="nf4").cuda()
    assert set(sd) == set(lin.state_dict())
    rebuilt = GroupedLinear4bit(E, K, N, bias=True, compress_statistics=nested, quant_type="nf4")
    rebuilt.weight = Params4bit.from_prequantized(
        sd["weight"], {k[len("weight."):]: v for k, v in sd.items() if k.startswith("weight.")}, device="cuda",
        module=rebuilt)
    rebuilt.bias = torch.nn.Parameter(sd["bias"].cuda())
    with torch.no_grad():
        assert torch.equal(rebuilt(x, offs), y)


# ---------------------------------------------------------------------------------------------------- real sizes
def _routed(M_tokens, E, topk, seed):
    """Seeded top-k routing of M_tokens tokens: the expert-sorted row counts (M_tokens * topk rows)."""
    g = torch.Generator().manual_seed(seed)
    choice = torch.rand(M_tokens, E, generator=g).topk(topk, dim=1).indices.reshape(-1)
    return torch.bincount(choice, minlength=E).tolist()


def test_qwen3_30b_a3b_gate_up_top8_bit_for_bit():
    E, N, K = 128, 1536, 2048
    counts = _routed(512, E, 8, seed=3)
    offs, M = routing(counts)
    qW, qs = _expert_weight(E, N, K, nested=True, seed=3)
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    p = dict(x=x, packed=qW, absmax=qs.state2.absmax, absmax_8bit=qs.absmax, absmax_code=qs.state2.code,
             absmax_offset=qs.offset.reshape(1).float(), M=M, N=E * N, K=K, bs=qs.blocksize, qt="nf4", dtype="bf16",
             bias=None)
    mt = rule_tile(M, E)
    got, buf = grouped_mt(p, E, offs, mt)
    check_grouped(p, E, offs, mt, got, buf, oracle=False)


def test_mixtral_8x7b_w1_w3_top2_against_the_oracle():
    import oracle

    E, N, K = 8, 28672, 4096
    counts = _routed(1024, E, 2, seed=4)
    offs, M = routing(counts)
    qW, qs = _expert_weight(E, N, K, nested=False, seed=4)
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    p = dict(x=x, packed=qW, absmax=qs.absmax, absmax_8bit=None, absmax_code=None, absmax_offset=None, M=M, N=E * N,
             K=K, bs=qs.blocksize, qt="nf4", dtype="bf16", bias=None)
    got, _ = grouped_mt(p, E, offs, 0, entry="prod")
    rows = np.random.default_rng(4).choice(M, 6, replace=False)
    packed = qW.cpu().numpy().reshape(-1)
    absmax = qs.absmax.cpu().numpy()
    per_e = N * K
    for m in rows:
        e = int(np.searchsorted(offs, m, side="right"))
        xb = oracle.widen(nat.to_bits(x[m:m + 1]), "bf16")
        y64 = oracle.gemm_4bit(xb, packed[e * per_e // 2:(e + 1) * per_e // 2],
                               absmax[e * per_e // qs.blocksize:(e + 1) * per_e // qs.blocksize], 1, N, K,
                               qs.blocksize, "nf4", "bf16")
        assert_close_to_exact(got[m:m + 1], y64, "bf16", K)
