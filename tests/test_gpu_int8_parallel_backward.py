"""GPU tests of the tensor-parallel LLM.int8() backward: the one-pass dequantisation of the int8 weight against the
torch expression of ``MatMul8bitLt.backward`` (bit for bit), then the column and row layers' input gradients at worlds
of 1, 2, 4 and 8 (the ranks simulated in turn on one GPU, running the layers' own forward and backward), their
relations to each other and to the unsharded ``Linear8bitLt``, outlier columns, gradient layouts and one LoRA step."""
import pytest
import torch

from tests import _native as nat
from tests.test_gpu_gemm4 import assert_close_to_exact
from tests.test_gpu_int8_parallel import _col_layers, _outlier_cols, _reference, _row_layers
from tests.test_gpu_parallel_backward import _SimWorld, _bits, _fwd_bwd, _leaf

pytestmark = pytest.mark.gpu

_NAME = {torch.bfloat16: "bf16", torch.float16: "fp16"}


def _torch_weight(CB, SCB, dtype):
    """The weight exactly as ``MatMul8bitLt.backward`` builds it."""
    return CB.to(dtype, copy=True).mul_(SCB.unsqueeze(1).mul(1.0 / 127.0))


class _SimWorld8(_SimWorld):
    """:class:`_SimWorld` with the all-reduce MAX the int8 layers' forward runs (row statistics, outlier flags)."""

    def __init__(self, world, monkeypatch):
        super().__init__(world, monkeypatch)
        import bitsandbytes_b200.parallel as par

        monkeypatch.setattr(par.dist, "all_reduce", self.all_reduce)

    def all_reduce(self, t, op=None, group=None):
        import torch.distributed as dist

        assert op == dist.ReduceOp.MAX
        self._exchange(t.clone(), lambda r: t.copy_(torch.stack(self.slots).amax(0)))


# ------------------------------------------------------------------------------------------------------ the kernel
def _codes(rows, cols, seed):
    g = torch.Generator().manual_seed(seed)
    CB = torch.randint(-128, 128, (rows, cols), generator=g, dtype=torch.int8)
    CB.view(-1)[::7] = 127
    CB.view(-1)[3::11] = -127
    CB.view(-1)[5::13] = -128
    SCB = torch.rand(rows, generator=g) * 4.0 + 1e-3
    SCB[1::5] = 0.0          # an all-zero weight row
    SCB[2::9] = 3e-37        # products below the fp32 normal range
    SCB[3::9] = 1e5          # products above the fp16 range
    return CB.cuda(), SCB.cuda()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("rows,cols,pad,offset", [
    (1, 1, 0, 0), (3, 7, 0, 0), (37, 100, 0, 0), (64, 1024, 0, 0), (17, 1000, 8, 0), (33, 4109, 5, 0),
    (9, 96, 3, 0), (21, 256, 0, 1), (12, 130, 6, 3), (3584, 8192, 0, 0)])
def test_dequant_rows_equals_the_torch_expression(dtype, rows, cols, pad, offset):
    """Bit for bit the torch expression, for every column count (16-code vectors with a scalar head and tail, or all
    scalar), row pitches ``ldo > cols`` (the NaN sentinels between rows stay NaN), unaligned codes and outputs
    (``offset`` elements into their storage), zero rows, codes at +-127 and -128, and products that leave the normal
    range of fp32 or the range of fp16."""
    from bitsandbytes_b200.backends.cuda import int8_dequant_rows

    CB, SCB = _codes(rows, cols, seed=rows * cols + pad)
    if offset:
        CB = torch.cat([torch.zeros(offset, dtype=torch.int8, device="cuda"), CB.view(-1)])[offset:].view(rows, cols)
    buf = torch.full((rows * (cols + pad) + offset,), float("nan"), device="cuda", dtype=dtype)
    out = buf[offset:].view(rows, cols + pad)[:, :cols]
    assert int8_dequant_rows(CB, SCB, dtype, out=out) is out
    torch.cuda.synchronize()
    nat.check()
    assert torch.equal(_bits(out), _bits(_torch_weight(CB, SCB, dtype)))
    assert torch.isnan(buf[offset:].view(rows, cols + pad)[:, cols:].float()).all()
    assert torch.isnan(buf[:offset].float()).all()
    assert torch.equal(_bits(int8_dequant_rows(CB, SCB, dtype)), _bits(out))


def test_dequant_rows_return_codes_write_nothing():
    """fp32 (and any other dtype) returns 100, bad arguments 1 with the error message set; neither writes."""
    rows, cols = 8, 64
    CB, SCB = _codes(rows, cols, seed=1)

    def call(dtype_id, ldo=cols, r=rows, c=cols):
        out = torch.full((rows, cols), float("nan"), device="cuda")
        rc = nat.lib.cbnb_b200_int8_dequant_rows(CB.data_ptr(), SCB.data_ptr(), out.data_ptr(), ldo, r, c, dtype_id,
                                                 nat.stream())
        torch.cuda.synchronize()
        return rc, out

    for dtype_id in (0, 3, -1):
        rc, out = call(dtype_id)
        assert rc == 100 and torch.isnan(out).all()
    for kw in (dict(ldo=cols - 1), dict(r=-1), dict(c=-1)):
        rc, out = call(2, **kw)
        assert rc == 1 and torch.isnan(out).all(), kw
        with pytest.raises(RuntimeError, match="int8_dequant_rows"):
            nat.check()
    assert call(2, r=0)[0] == 0 and call(1, c=0)[0] == 0


# ------------------------------------------------------------------------------------------------------ the layers
def _layers(CB, SCB, bias, world, threshold, mode):
    from bitsandbytes_b200.parallel import (ColumnParallelLinear8bitLt, RowParallelLinear8bitLt, slice_int8_weight,
                                            slice_int8_weight_k)

    N, K = CB.shape
    if mode == "col":
        return _col_layers(CB, SCB, bias, world, threshold)
    if mode == "col_sp":
        return [ColumnParallelLinear8bitLt(slice_int8_weight(CB, SCB, world, r), N, bias, threshold=threshold,
                                           gather_output=False, sequence_parallel=True) for r in range(world)]
    if mode == "row":
        return _row_layers(CB, SCB, bias, world, threshold)
    return [RowParallelLinear8bitLt(slice_int8_weight_k(CB, SCB, world, r), K, bias, threshold=threshold,
                                    sequence_parallel=True) for r in range(world)]


def _run(monkeypatch, layers, x, gy, mode):
    """[(y, x.grad)] of every rank's own forward and backward: the column layer on the replicated x and gradient of the
    gathered output (col) or on its tokens and the gradient of its columns (col_sp); the row layer on the whole
    replicated x (row) or on its input features with the gradient of its tokens (row_sp)."""
    world = len(layers)
    Ms, rows, kr = x.shape[0] // world, layers[0].shard.rows, layers[0].shard.K

    def rank(r):
        L = layers[r]
        if mode == "col":
            return _fwd_bwd(L, x, gy)
        if mode == "col_sp":
            return _fwd_bwd(L, x[r * Ms:(r + 1) * Ms], gy[:, r * rows:(r + 1) * rows].contiguous())
        if mode == "row":
            return _fwd_bwd(L, x, gy)
        return _fwd_bwd(L, x[:, r * kr:(r + 1) * kr], gy[r * Ms:(r + 1) * Ms])

    return _SimWorld8(world, monkeypatch).run(rank)


def _unsharded_grad(lin, x, gy):
    xl = _leaf(x)
    lin(xl).backward(gy)
    return xl.grad


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("M", [1, 64, 2048])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("with_bias", [False, True])
def test_gradients_within_the_float64_bound(monkeypatch, world, M, dtype, with_bias):
    """Both layers through their own forward and backward: within the float64 bound of G . W (W the dequantised weight
    in T, exact in float64), as is the unsharded Linear8bitLt's x.grad; every rank holds the same column gradient, and
    the whole-input row gradient is the ranks' columns in rank order.  Under sequence parallelism (M divisible by the
    world) the column layer's rank r holds rows [r M/w, (r+1) M/w) of that gradient and the row layer its columns, bit
    for bit, and the forward outputs are the non-SP ones."""
    x, lin, _, CB, SCB, bias = _reference(M, dtype, with_bias, 0.0, seed=world * 100 + M)
    N, K = CB.shape
    gy = torch.randn(M, N, generator=torch.Generator().manual_seed(M + 5)).to(dtype).cuda()
    y64 = (gy.double() @ _torch_weight(CB, SCB, dtype).double()).cpu().numpy()
    assert_close_to_exact(_unsharded_grad(lin, x, gy), y64, _NAME[dtype], N)
    col = _run(monkeypatch, _layers(CB, SCB, bias, world, 0.0, "col"), x, gy, "col")
    row = _run(monkeypatch, _layers(CB, SCB, bias, world, 0.0, "row"), x, gy, "row")
    nat.check()
    want_col, want_row = col[0][1], row[0][1]
    assert_close_to_exact(want_col, y64, _NAME[dtype], N)
    assert_close_to_exact(want_row, y64, _NAME[dtype], N)
    for r in range(world):
        assert torch.equal(_bits(col[r][1]), _bits(want_col)), f"column rank {r}"
        assert torch.equal(_bits(row[r][1]), _bits(want_row)), f"row rank {r}"
    if M % world:
        return
    Ms, rows, kr = M // world, N // world, K // world
    col_sp = _run(monkeypatch, _layers(CB, SCB, bias, world, 0.0, "col_sp"), x, gy, "col_sp")
    row_sp = _run(monkeypatch, _layers(CB, SCB, bias, world, 0.0, "row_sp"), x, gy, "row_sp")
    nat.check()
    for r in range(world):
        assert torch.equal(_bits(col_sp[r][1]), _bits(want_col[r * Ms:(r + 1) * Ms])), f"column SP rank {r}"
        assert torch.equal(_bits(row_sp[r][1]), _bits(want_row[:, r * kr:(r + 1) * kr])), f"row SP rank {r}"
        assert torch.equal(col_sp[r][0], col[r][0][:, r * rows:(r + 1) * rows]), f"column SP forward rank {r}"
        assert torch.equal(row_sp[r][0], row[r][0][r * Ms:(r + 1) * Ms]), f"row SP forward rank {r}"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("threshold,J", [(0.0, 0), (6.0, 5), (6.0, 80)])
def test_world_one_through_autograd(dtype, threshold, J):
    """Through the layers' own forward at world 1: the output has a grad_fn, its bits are those of the no_grad call,
    and x.grad is T(torch.mm(G, W, out_dtype=fp32)) for the column layer and the unsharded Linear8bitLt's x.grad (the
    same cuBLAS call on the same operands) for the row layer, with or without outlier columns."""
    from bitsandbytes_b200.parallel import ColumnParallelLinear8bitLt, RowParallelLinear8bitLt

    cols = _outlier_cols(J, "spread") if J else ()
    x, lin, y_ref, CB, SCB, _ = _reference(96, dtype, True, threshold, cols, seed=J + 3)
    gy = torch.randn(y_ref.shape, generator=torch.Generator().manual_seed(J)).to(dtype).cuda()
    W = _torch_weight(CB, SCB, dtype)
    want = {"col": torch.mm(gy, W, out_dtype=torch.float32).to(dtype), "row": _unsharded_grad(lin, x, gy)}
    for kind, cls in (("col", ColumnParallelLinear8bitLt), ("row", RowParallelLinear8bitLt)):
        layer = cls.from_linear8bitlt(lin)
        xl = _leaf(x)
        y = layer(xl)
        assert y.grad_fn is not None
        with torch.no_grad():
            assert torch.equal(_bits(y), _bits(layer(x)))
        assert torch.equal(_bits(y), _bits(y_ref))
        y.backward(gy)
        assert torch.equal(_bits(xl.grad), _bits(want[kind])), kind


@pytest.mark.parametrize("J", [5, 80])
@pytest.mark.parametrize("world", [1, 4])
def test_outlier_columns_leave_the_gradient_alone(monkeypatch, J, world):
    """With outlier columns in x (up to 64: the GEMM epilogue's outlier term; past 64: the addmm chain) the gradient is
    the threshold-0 gradient bit for bit, on every rank of both layers, and the backward makes no host
    synchronisation."""
    x, _, _, CB, SCB, bias = _reference(64, torch.bfloat16, True, 6.0, _outlier_cols(J, "spread"), seed=J)
    gy = torch.randn(64, CB.shape[0], generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).cuda()
    for mode in ("col", "row"):  # one rank, in this thread: the backward alone under the synchronisation check
        layer = _layers(CB, SCB, bias, 1, 6.0, mode)[0]
        layer(x)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            layer._backward(gy, x.shape)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    for mode in ("col", "row"):
        got = _run(monkeypatch, _layers(CB, SCB, bias, world, 6.0, mode), x, gy, mode)
        want = _run(monkeypatch, _layers(CB, SCB, bias, world, 0.0, mode), x, gy, mode)
        for r in range(world):
            assert torch.equal(_bits(got[r][1]), _bits(want[r][1])), f"{mode} rank {r}"


@pytest.mark.parametrize("loss", ["sum", "mean0", "transposed"])
def test_backward_takes_the_gradient_layouts_autograd_produces(monkeypatch, loss):
    """`.sum()` hands the layers an expanded gradient, `.mean(0)` a broadcast one, a transposed use a column-major one.
    Through autograd at world 1 (bf16 and fp16), and through ``_backward`` at world 2: x.grad equals the gradient of
    the same loss passed in contiguous, for both layers."""
    M = 64
    f = {"sum": lambda y, v: y.sum(), "mean0": lambda y, v: y.mean(0).sum(),
         "transposed": lambda y, v: (y.t() @ v).float().sum()}[loss]
    for dtype in (torch.bfloat16, torch.float16):
        x, _, _, CB, SCB, bias = _reference(M, dtype, True, 0.0, seed=31)
        v = torch.randn(M, generator=torch.Generator().manual_seed(33)).to(dtype).cuda()
        for mode in ("col", "row"):
            layer = _layers(CB, SCB, bias, 1, 0.0, mode)[0]
            a, b = _leaf(x), _leaf(x)
            f(layer(a), v).backward()
            yd = layer(b).detach().requires_grad_()
            gy, = torch.autograd.grad(f(yd, v), yd)
            layer(b).backward(gy.contiguous())
            assert a.grad is not None and torch.equal(_bits(a.grad), _bits(b.grad)), (dtype, mode)
    x, _, _, CB, SCB, bias = _reference(M, torch.bfloat16, True, 0.0, seed=31)
    v = torch.randn(M, generator=torch.Generator().manual_seed(33)).to(torch.bfloat16).cuda()
    layers = {mode: _layers(CB, SCB, bias, 2, 0.0, mode) for mode in ("col", "row")}

    def step(r):
        out = []
        for mode in ("col", "row"):
            with torch.no_grad():
                y = layers[mode][r](x)
            yd = y.requires_grad_()
            gy, = torch.autograd.grad(f(yd, v), yd)
            out.append((layers[mode][r]._backward(gy, x.shape), layers[mode][r]._backward(gy.contiguous(), x.shape)))
        return out

    for res in _SimWorld8(2, monkeypatch).run(step):
        for got, want in res:
            assert torch.equal(got, want)


def _chain64(x, A, B, z, W1, W2, y):
    """Float64 gradients of the LoRA adapter (A, B) of loss = mean(y^2), y = W2 . silu(z), z = W1 . h, h = x + x A^T
    B^T, taken at the forward values the layers produced (z, y): the exact backward of the computation that ran."""
    z, y = z.double(), y.double()
    gy = 2.0 * y / y.numel()
    gs = gy @ W2
    sig = torch.sigmoid(z)
    gz = gs * (sig * (1.0 + z * (1.0 - sig)))
    gh = gz @ W1
    xa = x.double() @ A.double().t()
    return (gh @ B.double()).t() @ x.double(), gh.t() @ xa


def test_lora_adapter_trains_through_a_column_row_pair(monkeypatch):
    """x -> LoRA adapter -> column layer (gather_output=False) -> SiLU -> row layer, one step at world 1 (autograd) and
    at a simulated world of 2 (every rank's adapter gradients): within the bound of the float64 backward of the same
    forward values, as are those of the same model built from unsharded Linear8bitLt layers.  Each gradient passes
    through about five bf16 roundings of O(1)-conditioned products, so the bound is a relative norm of 5 * 2^-8."""
    import bitsandbytes_b200 as bnb  # noqa: F401 -- registers the ops the Linear8bitLt layers run
    from bitsandbytes_b200.parallel import (ColumnParallelLinear8bitLt, RowParallelLinear8bitLt, slice_int8_weight,
                                            slice_int8_weight_k)

    dtype = torch.bfloat16
    K, H, M, rank_r = 1024, 2048, 256, 16
    _, lin1, _, CB1, SCB1, _ = _reference(M, dtype, False, 0.0, seed=21, N=H, K=K)
    _, lin2, _, CB2, SCB2, _ = _reference(M, dtype, False, 0.0, seed=22, N=K, K=H)
    W1, W2 = _torch_weight(CB1, SCB1, dtype).double(), _torch_weight(CB2, SCB2, dtype).double()
    g = torch.Generator().manual_seed(23)
    x = torch.randn(M, K, generator=g).to(dtype).cuda()
    A0 = (torch.randn(rank_r, K, generator=g) / K**0.5).to(dtype).cuda()
    B0 = (torch.randn(K, rank_r, generator=g) / rank_r**0.5).to(dtype).cuda()
    bound = 5 * 2.0**-8

    def check(grads, z, y):
        for got, want in zip(grads, _chain64(x, A0, B0, z, W1, W2, y)):
            assert got is not None and torch.isfinite(got).all()
            rel = float((got.double() - want).norm() / want.norm())
            assert rel < bound, rel

    def autograd_step(first, second):
        A, B = A0.clone().requires_grad_(), B0.clone().requires_grad_()
        h = x + (x @ A.t()) @ B.t()
        z = first(h)
        y = second(torch.nn.functional.silu(z))
        (y.float() ** 2).mean().backward()
        return (A.grad, B.grad), z.detach(), y.detach()

    check(*autograd_step(lin1, lin2))
    col = ColumnParallelLinear8bitLt(slice_int8_weight(CB1, SCB1, 1, 0), H, gather_output=False)
    row = RowParallelLinear8bitLt(slice_int8_weight_k(CB2, SCB2, 1, 0), H)
    check(*autograd_step(col, row))

    world = 2
    shards = [(slice_int8_weight(CB1, SCB1, world, r), slice_int8_weight_k(CB2, SCB2, world, r)) for r in range(world)]

    def rank(r):
        c = ColumnParallelLinear8bitLt(shards[r][0], H, gather_output=False)
        w = RowParallelLinear8bitLt(shards[r][1], H)
        A, B = A0.clone().requires_grad_(), B0.clone().requires_grad_()
        h = x + (x @ A.t()) @ B.t()
        with torch.no_grad():
            z = c(h)
            s = torch.nn.functional.silu(z)
            y = w(s)
        yd = y.clone().requires_grad_()
        gy, = torch.autograd.grad((yd.float() ** 2).mean(), yd)
        gs = w._backward(gy, s.shape)
        zd = z.clone().requires_grad_()
        gz, = torch.autograd.grad(torch.nn.functional.silu(zd), zd, gs)
        h.backward(c._backward(gz, h.shape))
        return (A.grad, B.grad), z, y

    res = _SimWorld8(world, monkeypatch).run(rank)
    z = torch.cat([res[r][1] for r in range(world)], dim=1)
    for r in range(world):
        assert torch.equal(res[r][2], res[0][2]), f"rank {r} output"
        assert all(torch.equal(a, b) for a, b in zip(res[r][0], res[0][0])), f"rank {r} adapter gradients"
    check(res[0][0], z, res[0][2])
