"""GPU: the grouped LLM.int8() GEMM (every expert of a mixture-of-experts layer in one launch) through the op,
bnb.grouped_matmul_8bit and bnb.nn.GroupedLinear8bitLt.

Each expert's rows must equal, bit for bit, the device-side route on that expert's rows alone -- int8_mixed_mm_flags
with the expert's own outlier flags, or int8_scaled_mm at threshold 0 -- and, up to 64 outlier columns, the eager
int8_mixed_scaled_mm of Linear8bitLt.  Rows past the last clamped end must be exactly +0, and every row must be within
a bound of a float64 oracle.  The outliers are planted so that the experts' sets differ: none, a few, exactly 64 and
80 (past the 64 columns the operands hold), and one that only a single-row expert has.
"""
import pytest
import torch

import bitsandbytes_b200 as bnb
import bitsandbytes_b200.functional as F
from bitsandbytes_b200.backends.cuda import int8_grouped_mm, int8_mixed_mm_flags, int8_vectorwise_quant_flags
from bitsandbytes_b200.nn import GroupedLinear8bitLt, Linear8bitLt

pytestmark = pytest.mark.gpu

DEV = "cuda"
THR = 6.0


def clamped_ends(offs, M):
    ends, run = [], 0
    for o in offs:
        run = min(max(run, o), M)
        ends.append(run)
    return ends


def expert_weight(E, N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    W = torch.randn(E, N, K, device=DEV, generator=g) / K**0.5
    CB, SCB, _ = F.int8_vectorwise_quant(W.to(torch.float16))
    return CB, SCB


def activations(M, K, ends, dtype, seed, plant=True):
    """Seeded activations below the threshold, with per-expert outlier columns planted when ``plant``: expert e gets
    none, 80, 64 or 3 columns by e % 4 (set in one of its rows), and a single-row expert a column of its own."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    A = (torch.rand(M, K, device=DEV, generator=g) * 2 - 1) * 4
    if plant:
        gc = torch.Generator().manual_seed(seed)
        begin = 0
        for e, end in enumerate(ends):
            rows = end - begin
            if rows > 0:
                n = (0, 80, 64, 3)[e % 4] if rows > 1 else 1
                cols = torch.randperm(K, generator=gc)[:n].to(DEV)
                r = begin + int(torch.randint(rows, (1,), generator=gc))
                A[r, cols] = 7.0 + torch.rand(n, device=DEV, generator=g)
                A[r, cols[::2]] *= -1
            begin = end
    return A.to(dtype)


def per_expert(A, CB, SCB, ends, threshold, bias):
    """Each expert's rows through the single-expert device route on those rows alone."""
    E, N, K = CB.shape
    outs, begin = [], 0
    for e, end in enumerate(ends):
        if end > begin:
            Ae = A[begin:end]
            b = bias[e] if bias is not None else None
            CA, SCA, flags = int8_vectorwise_quant_flags(Ae.to(torch.float16), threshold)
            if threshold > 0:
                y = int8_mixed_mm_flags(Ae, CA, CB[e], SCA, SCB[e * N:(e + 1) * N], flags, b)
            else:
                y = torch.ops.bitsandbytes.int8_scaled_mm(CA, CB[e], SCA, SCB[e * N:(e + 1) * N], bias=b, dtype=A.dtype)
            outs.append((e, begin, end, y, int(flags.sum()) if flags is not None else 0))
        begin = end
    return outs


def eager(Ae, CBe, SCBe, threshold, b):
    """The eager Linear8bitLt forward (MatMul8bitLt): nonzero outlier list, int8_mixed_scaled_mm."""
    CA, SCA, cols = F.int8_vectorwise_quant(Ae.to(torch.float16), threshold=threshold)
    if threshold > 0:
        return torch.ops.bitsandbytes.int8_mixed_scaled_mm(Ae, CA, CBe, SCA, SCBe, cols, b)[0]
    return torch.ops.bitsandbytes.int8_scaled_mm(CA, CBe, SCA, SCBe, bias=b, dtype=Ae.dtype)


def bits(t):
    return t.contiguous().view(torch.int16)


def assert_bits(got, want, what):
    diff = (bits(got) != bits(want)).sum().item()
    assert diff == 0, f"{what}: {diff} elements differ in their bits"


def check_against_float64(got, A, CB, SCB, ends, threshold, bias):
    """|got - y64| within the int8 rounding of the non-outlier entries, the 16-bit rounding of the outlier weights and
    of the result, where y64 = A . W^T + bias in float64 with W = CB * SCB / 127, for the routed rows."""
    E, N, K = CB.shape
    W = CB.double() * (SCB.double().view(E, N, 1) / 127)
    Ad = A.double()
    begin = 0
    for e, end in enumerate(ends):
        if end > begin:
            a = Ad[begin:end]
            y = a @ W[e].T + (bias[e].double() if bias is not None else 0)
            small = a.abs() < threshold if threshold > 0 else torch.ones_like(a, dtype=torch.bool)
            sca = torch.where(small, a.abs(), torch.zeros_like(a)).amax(1, keepdim=True)
            bound = sca / 254 * W[e].abs().sum(1) + 2**-7 * (a.abs() @ W[e].abs().T) + 2**-9 * y.abs() + 1e-3
            err = (got[begin:end].double() - y).abs()
            assert bool((err <= bound).all()), f"expert {e}: max excess {(err - bound).max().item()}"
        begin = end


ROUTINGS = {
    # name: (offs, M)
    "ragged": ([37, 45, 187, 188, 388, 400], 400),
    "empty_experts": ([0, 0, 90, 90, 90, 90], 90),
    "one_expert": ([0, 0, 0, 300, 300, 300], 300),
    "single_rows": ([1, 2, 3, 4, 5, 6], 6),
    "tail_rows": ([20, 50, 50, 55, 95, 96], 121),
    "malformed": ([50, 20, -5, 400, 100, 90], 200),
}


@pytest.mark.parametrize("routing", list(ROUTINGS))
@pytest.mark.parametrize("threshold", [0.0, THR])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_every_instance_and_routing(dtype, threshold, routing):
    offs, M = ROUTINGS[routing]
    E, N, K = len(offs), 320, 512
    ends = clamped_ends(offs, M)
    CB, SCB = expert_weight(E, N, K, seed=1)
    A = activations(M, K, ends, dtype, seed=2, plant=threshold > 0)
    bias = (torch.randn(E, N, device=DEV) * 0.1).to(dtype)
    offs_t = torch.tensor(offs, dtype=torch.int32, device=DEV)
    got = int8_grouped_mm(A, CB, SCB, offs_t, threshold, bias)
    counts = []
    for e, begin, end, want, J in per_expert(A, CB, SCB, ends, threshold, bias):
        assert_bits(got[begin:end], want, f"rows [{begin}, {end})")
        counts.append(J)
        if J <= 64:
            assert_bits(got[begin:end], eager(A[begin:end], CB[e], SCB[e * N:(e + 1) * N], threshold, bias[e]),
                        f"rows [{begin}, {end}) against the eager Linear8bitLt")
    assert bool((bits(got[ends[-1]:]) == 0).all()), "tail rows must be +0"
    check_against_float64(got, A, CB, SCB, ends, threshold, bias)
    if threshold > 0 and routing == "ragged":
        assert 0 in counts and 80 in counts and 64 in counts and 1 in counts  # the planted sets reached the kernel


def test_outlier_only_in_a_single_row_expert_stays_its_own():
    """A column that only a one-row expert flags is neither zeroed in nor added to the other experts' rows."""
    E, N, K, M = 3, 256, 256, 41
    offs = [20, 21, 41]
    CB, SCB = expert_weight(E, N, K, seed=5)
    A = activations(M, K, offs, torch.bfloat16, seed=6, plant=False)
    A[20, 7] = 9.0
    got = int8_grouped_mm(A, CB, SCB, torch.tensor(offs, dtype=torch.int32, device=DEV), THR)
    for _, begin, end, want, J in per_expert(A, CB, SCB, offs, THR, None):
        assert J == (1 if begin == 20 else 0)
        assert_bits(got[begin:end], want, f"rows [{begin}, {end})")
    # without the single-row expert's column, the neighbours are the plain int8 result
    assert_bits(got[:20], eager(A[:20], CB[0], SCB[:N], 0.0, None), "expert 0 at no outliers")


def test_no_host_sync_at_threshold():
    E, N, K = 8, 256, 512
    offs, M = [10, 40, 40, 41, 100, 130, 131, 160], 170
    CB, SCB = expert_weight(E, N, K, seed=7)
    A = activations(M, K, offs, torch.bfloat16, seed=8)
    offs_t = torch.tensor(offs, dtype=torch.int32, device=DEV)
    bias = torch.zeros(E, N, dtype=torch.bfloat16, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = bnb.grouped_matmul_8bit(A, CB, SCB, offs_t, threshold=THR, bias=bias)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert out.shape == (M, N)


def test_cuda_graph_replays_new_routings_and_outlier_sets():
    E, N, K, M = 8, 384, 512, 256
    CB, SCB = expert_weight(E, N, K, seed=9)
    bias = (torch.randn(E, N, device=DEV) * 0.1).to(torch.bfloat16)
    cum = lambda c: torch.tensor(c).cumsum(0).tolist()  # noqa: E731
    routings = [cum([32] * E), cum([0, 100, 1, 0, 55, 30, 0, 60]), [256] * E, cum([3] * E), [90, 180, -4, 500, 10, 0, 0, 0]]
    offs = torch.tensor(routings[0], dtype=torch.int32, device=DEV)
    A = activations(M, K, routings[0], torch.bfloat16, seed=10)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(2):
            bnb.grouped_matmul_8bit(A, CB, SCB, offs, threshold=THR, bias=bias)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.no_grad():
        out = bnb.grouped_matmul_8bit(A, CB, SCB, offs, threshold=THR, bias=bias)
    for i, r in enumerate(routings[1:] + routings[:1]):
        ends = clamped_ends(r, M)
        offs.copy_(torch.tensor(r, dtype=torch.int32))
        A.copy_(activations(M, K, ends, torch.bfloat16, seed=20 + i))
        graph.replay()
        with torch.no_grad():
            want = bnb.grouped_matmul_8bit(A, CB, SCB, offs, threshold=THR, bias=bias)
        assert_bits(out, want, f"replay {i}")
        Js = [J for *_, J in per_expert(A, CB, SCB, ends, THR, bias)]
        if i == 0:
            assert max(Js) > 64  # a replay whose outlier count crosses the operands' 64 columns


@pytest.mark.parametrize("threshold", [0.0, THR])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_grouped_linear8bitlt_matches_linear8bitlt_modules(dtype, threshold):
    E, K, N = 4, 256, 192
    torch.manual_seed(11)
    g = GroupedLinear8bitLt(E, K, N, bias=True, threshold=threshold)
    W, b = g.weight.data.clone(), g.bias.data.clone()
    g = g.cuda()
    mods = []
    for e in range(E):
        m = Linear8bitLt(K, N, bias=True, has_fp16_weights=False, threshold=threshold)
        m.weight = bnb.nn.Int8Params(W[e].clone(), requires_grad=False, has_fp16_weights=False)
        m.bias = torch.nn.Parameter(b[e].clone())
        mods.append(m.cuda())
    assert torch.equal(g.weight.data.view(E * N, K), torch.cat([m.weight.data for m in mods]))
    counts = [30, 1, 57, 0]
    ends = torch.tensor(counts).cumsum(0).tolist()
    M = ends[-1] + 5
    x = activations(M, K, ends, dtype, seed=12, plant=threshold > 0)
    offs = torch.tensor(ends, dtype=torch.int32, device=DEV)
    with torch.no_grad():
        y = g(x, offs)
        begin = 0
        for e, end in enumerate(ends):
            if end > begin:
                assert_bits(y[begin:end], mods[e](x[begin:end]), f"expert {e}")
            begin = end
    assert bool((bits(y[ends[-1]:]) == 0).all())
    # the state dict round-trips, loaded before and after .cuda()
    sd = {k: v.cpu() for k, v in g.state_dict().items()}
    assert set(sd) == {"weight", "SCB", "weight_format", "bias"}
    before = GroupedLinear8bitLt(E, K, N, bias=True, threshold=threshold)
    before.load_state_dict(sd)
    before = before.cuda()
    after = GroupedLinear8bitLt(E, K, N, bias=True, threshold=threshold).cuda()
    after.load_state_dict(sd)
    with torch.no_grad():
        assert_bits(before(x, offs), y, "loaded before .cuda()")
        assert_bits(after(x, offs), y, "loaded after .cuda()")


@pytest.mark.parametrize("tail", [0, 7])
def test_autograd_bf16_against_float64(tail):
    E, N, K = 4, 256, 512
    counts = [40, 0, 1, 80]
    ends = torch.tensor(counts).cumsum(0).tolist()
    M = ends[-1] + tail
    CB, SCB = expert_weight(E, N, K, seed=13)
    A = activations(M, K, ends, torch.bfloat16, seed=14).requires_grad_(True)
    bias = (torch.randn(E, N, device=DEV) * 0.1).to(torch.bfloat16).requires_grad_(True)
    offs = torch.tensor(ends, dtype=torch.int32, device=DEV)
    out = bnb.grouped_matmul_8bit(A, CB, SCB, offs, threshold=THR, bias=bias)
    with torch.no_grad():
        assert_bits(out, bnb.grouped_matmul_8bit(A, CB, SCB, offs, threshold=THR, bias=bias), "forward")
    G = torch.randn(M, N, device=DEV).to(torch.bfloat16)
    out.backward(G)
    W = (CB.double() * (SCB.double().view(E, N, 1) / 127))
    Gd = G.double()
    gA = torch.zeros(M, K, dtype=torch.float64, device=DEV)
    bound = torch.full((M, K), 1e-3, dtype=torch.float64, device=DEV)
    gb = torch.zeros(E, N, dtype=torch.float64, device=DEV)
    begin = 0
    for e, end in enumerate(ends):
        gA[begin:end] = Gd[begin:end] @ W[e]
        # the weight rounded to bf16, fp32 sums, the result rounded to bf16
        bound[begin:end] += 2**-7 * (Gd[begin:end].abs() @ W[e].abs())
        gb[e] = Gd[begin:end].sum(0)
        begin = end
    err = (A.grad.double() - gA).abs()
    assert bool((err <= bound).all()), f"grad_A: max excess {(err - bound).max().item()}"
    assert bool((bits(A.grad[ends[-1]:]) == 0).all()), "tail rows get no gradient"
    assert torch.allclose(bias.grad.double(), gb, rtol=2**-7, atol=1e-2)


def test_fp16_training_is_refused():
    E, N, K = 2, 64, 64
    CB, SCB = expert_weight(E, N, K, seed=15)
    A = torch.randn(8, K, device=DEV, dtype=torch.float16, requires_grad=True)
    with pytest.raises(ValueError, match="bfloat16 only"):
        bnb.grouped_matmul_8bit(A, CB, SCB, torch.tensor([4, 8], dtype=torch.int32, device=DEV))


# ---------------------------------------------------------------------------------------------------- real sizes
def _routed(M_tokens, E, topk, seed):
    """Seeded top-k routing of M_tokens tokens: the expert-sorted clamped ends (M_tokens * topk rows)."""
    g = torch.Generator().manual_seed(seed)
    choice = torch.rand(M_tokens, E, generator=g).topk(topk, dim=1).indices.reshape(-1)
    return torch.bincount(choice, minlength=E).cumsum(0).tolist()


@pytest.mark.parametrize("name,E,N,K,topk,tokens", [
    ("mixtral_8x7b_w1_w3", 8, 28672, 4096, 2, 512),
    ("mixtral_8x7b_w2", 8, 4096, 14336, 2, 512),
    ("qwen3_30b_a3b_gate_up", 128, 1536, 2048, 8, 256),
    ("qwen3_30b_a3b_down", 128, 2048, 768, 8, 256),
])
def test_real_sizes_bit_for_bit(name, E, N, K, topk, tokens):
    ends = _routed(tokens, E, topk, seed=16)
    M = ends[-1]
    CB, SCB = expert_weight(E, N, K, seed=17)
    A = activations(M, K, ends, torch.bfloat16, seed=18)
    got = int8_grouped_mm(A, CB, SCB, torch.tensor(ends, dtype=torch.int32, device=DEV), THR)
    for _, begin, end, want, _ in per_expert(A, CB, SCB, ends, THR, None):
        assert_bits(got[begin:end], want, f"{name} rows [{begin}, {end})")
    check_against_float64(got, A, CB, SCB, ends, THR, None)
