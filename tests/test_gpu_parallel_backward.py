"""GPU tests of the backward of the tensor-parallel Linear4bit layers: their gradients at worlds of 1, 2, 4 and 8 (the
ranks simulated in turn on one GPU), rank agreement, the sequence-parallel rows, the layers' own forward and backward
through simulated collectives, the gradient layouts autograd produces, and one training step of a LoRA adapter in front
of a column -> row pair."""
import pytest
import torch

from tests import _native as nat
from tests.test_gpu_gemm4 import assert_close_to_exact

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


# ------------------------------------------------------------------------------------------------------ the layers
def _model(N, K, dtype, nested, seed):
    import bitsandbytes_b200.functional as F

    g = torch.Generator().manual_seed(seed)
    W = (torch.randn(N, K, generator=g) / K**0.5).to(dtype).cuda()
    qW, qs = F.quantize_4bit(W, blocksize=64, quant_type="nf4", compress_statistics=nested)
    return qW, qs, F.dequantize_4bit(qW, qs).double()


def _unsharded_grad(x_shape, qW, qs, grad_y):
    """The single-GPU Linear4bit backward (dequantise + cuBLAS) for the output gradient grad_y."""
    import bitsandbytes_b200 as bnb

    x = torch.zeros(x_shape, device="cuda", dtype=grad_y.dtype, requires_grad=True)
    bnb.matmul_4bit(x, qW.t(), qs).backward(grad_y)
    return x.grad


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("M", [1, 64, 2048])
@pytest.mark.parametrize("dtype,nested", [(torch.bfloat16, False), (torch.float16, True)])
def test_column_layer_gradient(world, M, dtype, nested):
    """Every rank's partial of the gathered-output layer reduced in rank order: the same bits on every rank, the bits of
    the gather_output=False layer (its own contiguous columns), within the float64 bound of the unsharded backward,
    and, per rank of a sequence-parallel world, rows [r M/w, (r+1) M/w) of that result."""
    from bitsandbytes_b200.backends.cuda import reduce_partials
    from bitsandbytes_b200.parallel import ColumnParallelLinear4bit, slice_quantized_weight

    N, K = 2048, 1024
    qW, qs, W64 = _model(N, K, dtype, nested, seed=world + M)
    gy = torch.randn(M, N, generator=torch.Generator().manual_seed(M)).to(dtype).cuda()
    shards = [slice_quantized_weight(qW, qs, world, r) for r in range(world)]
    gathered = [ColumnParallelLinear4bit(s, N) for s in shards]
    local = [ColumnParallelLinear4bit(s, N, gather_output=False) for s in shards]
    stage = torch.full((world, M, K), float("nan"), device="cuda")
    for r, L in enumerate(gathered):
        L.input_grad_partial(gy, stage[r])
    grad = [reduce_partials(stage, dtype) for _ in range(world)]
    stage2 = torch.full_like(stage, float("nan"))
    for r, L in enumerate(local):
        L.input_grad_partial(gy[:, L.shard.row0:L.shard.row0 + L.shard.rows].contiguous(), stage2[r])
    torch.cuda.synchronize()
    nat.check()
    assert torch.equal(stage2.view(torch.int32), stage.view(torch.int32))
    for r in range(world):
        assert torch.equal(_bits(grad[r]), _bits(grad[0])), f"rank {r}"
    if world == 1:
        assert torch.equal(_bits(grad[0]), _bits(stage[0].to(dtype)))
    dt = "bf16" if dtype == torch.bfloat16 else "fp16"
    y64 = (gy.double() @ W64).cpu().numpy()
    assert_close_to_exact(grad[0], y64, dt, N)
    assert_close_to_exact(_unsharded_grad((M, K), qW, qs, gy), y64, dt, N)
    if M % world == 0:
        Ms = M // world
        for r in range(world):
            sp = reduce_partials(stage[:, r * Ms:(r + 1) * Ms].contiguous(), dtype)
            assert torch.equal(_bits(sp), _bits(grad[0][r * Ms:(r + 1) * Ms])), f"SP rank {r}"


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("M", [1, 64, 2048])
def test_row_layer_gradient(world, M):
    """grad_x_r = grad_y . dequant(W_r) for every rank: its columns of the unsharded input gradient within the float64
    bound; under sequence parallelism the gathered token rows give the same input."""
    from bitsandbytes_b200.parallel import RowParallelLinear4bit, slice_quantized_weight_k

    dtype = torch.bfloat16
    N, K = 1536, 4096
    qW, qs, W64 = _model(N, K, dtype, True, seed=world * M)
    gy = torch.randn(M, N, generator=torch.Generator().manual_seed(M + 1)).to(dtype).cuda()
    layers = [RowParallelLinear4bit(slice_quantized_weight_k(qW, qs, world, r), K) for r in range(world)]
    grad = torch.cat([L.input_grad(gy) for L in layers], dim=1)
    torch.cuda.synchronize()
    nat.check()
    y64 = (gy.double() @ W64).cpu().numpy()
    assert_close_to_exact(grad, y64, "bf16", N)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_autograd_reaches_the_input_at_world_one(dtype):
    """Through the layers' own forward: the output has a grad_fn and x.grad is T(P_0) of the fp32 partial (column
    layer, 16-bit) or the rounded product (row layer, and fp32); the forward's bits are those of the inference call."""
    from bitsandbytes_b200.parallel import ColumnParallelLinear4bit, RowParallelLinear4bit, input_grad_dequant_matmul

    N, K, M = 1024, 768, 96
    qW, qs, _ = _model(N, K, dtype, False, seed=11)
    g = torch.Generator().manual_seed(12)
    col = ColumnParallelLinear4bit.from_quantized(qW, qs)
    row = RowParallelLinear4bit.from_quantized(qW, qs)
    for layer, shape in ((col, (2, M // 2, K)), (row, (2, M // 2, K))):
        x = torch.randn(*shape, generator=g).to(dtype).cuda().requires_grad_()
        y = layer(x)
        with torch.no_grad():
            assert torch.equal(y, layer(x.detach()))
        assert y.grad_fn is not None
        gy = torch.randn(y.shape, generator=g).to(dtype).cuda()
        y.backward(gy)
        G = gy.reshape(M, N)
        if layer is col and dtype != torch.float32:
            want = input_grad_dequant_matmul(G, layer.shard, torch.float32).to(dtype)  # T(P_0)
        else:
            want = input_grad_dequant_matmul(G, layer.shard, dtype)
        assert x.grad is not None and x.grad.shape == x.shape
        assert torch.equal(_bits(x.grad.reshape(M, K)), _bits(want))


@pytest.mark.parametrize("nested", [False, True])
def test_lora_adapter_trains_through_a_column_row_pair(nested):
    """x -> LoRA adapter -> column layer (gather_output=False) -> row layer, one step: the adapter's gradients match
    those of the same model on the single-GPU matmul_4bit."""
    import bitsandbytes_b200 as bnb
    from bitsandbytes_b200.parallel import ColumnParallelLinear4bit, RowParallelLinear4bit

    dtype = torch.bfloat16
    K, H, M, r = 1024, 2816, 256, 16
    q1, s1, _ = _model(H, K, dtype, nested, seed=21)
    q2, s2, _ = _model(K, H, dtype, nested, seed=22)
    g = torch.Generator().manual_seed(23)
    x = torch.randn(M, K, generator=g).to(dtype).cuda()
    A0 = (torch.randn(r, K, generator=g) / K**0.5).to(dtype).cuda()
    B0 = (torch.randn(K, r, generator=g) / r**0.5).to(dtype).cuda()
    col = ColumnParallelLinear4bit.from_quantized(q1, s1, gather_output=False)
    row = RowParallelLinear4bit.from_quantized(q2, s2)

    def step(first, second):
        A, B = A0.clone().requires_grad_(), B0.clone().requires_grad_()
        h = x + (x @ A.t()) @ B.t()
        y = second(torch.nn.functional.silu(first(h)))
        (y.float() ** 2).mean().backward()
        return A.grad, B.grad

    got = step(col, row)
    want = step(lambda h: bnb.matmul_4bit(h, q1.t(), s1), lambda h: bnb.matmul_4bit(h, q2.t(), s2))
    for a, b in zip(got, want):
        assert a is not None and torch.isfinite(a).all()
        rel = float((a.float() - b.float()).norm() / b.float().norm())
        assert rel < 1e-2, rel


# ------------------------------------------------------------------------------------------- simulated collectives
class _SimWorld:
    """`world` ranks as threads on one GPU, running the layers' own forward and ``_backward`` (called directly: autograd
    runs every CUDA backward on one engine thread per device, where the ranks' collectives would wait for each other
    forever), the collectives exchanging the ranks' real tensors.  Only one rank runs between two collectives (a lock handed over at each of them), because the
    library's per-stream workspace is shared by every thread that launches on the one stream."""

    def __init__(self, world, monkeypatch):
        import threading

        import bitsandbytes_b200.parallel as par

        self.world, self.local = world, threading.local()
        self.lock, self.barrier = threading.Lock(), threading.Barrier(world, timeout=300)
        self.slots = [None] * world
        monkeypatch.setattr(par, "_group_world_rank", lambda group: (world, self.local.rank))
        monkeypatch.setattr(par.dist, "all_gather_into_tensor", self.all_gather_into_tensor)
        monkeypatch.setattr(par.dist, "all_to_all_single", self.all_to_all_single)

    def _exchange(self, inp, read):
        self.slots[self.local.rank] = inp
        for step in (lambda: None, lambda: read(self.local.rank)):
            step()
            self.lock.release()
            self.barrier.wait()
            self.lock.acquire()

    def all_gather_into_tensor(self, out, inp, group=None):
        self._exchange(inp, lambda r: out.view(self.world, -1).copy_(torch.stack([s.reshape(-1) for s in self.slots])))

    def all_to_all_single(self, out, inp, group=None):
        def read(r):
            for s in range(self.world):
                out.view(self.world, -1)[s].copy_(self.slots[s].reshape(self.world, -1)[r])
        self._exchange(inp, read)

    def run(self, fn):
        """[fn(rank) for every rank], the ranks run as threads."""
        import threading

        results, errors = [None] * self.world, []

        def body(r):
            self.local.rank = r
            torch.cuda.synchronize()  # makes the primary context current in this thread, for the library's driver calls
            self.lock.acquire()
            try:
                results[r] = fn(r)
            except BaseException as e:  # noqa: BLE001 -- re-raised below, the other ranks released
                errors.append(e)
                self.barrier.abort()
            finally:
                self.lock.release()

        threads = [threading.Thread(target=body, args=(r,)) for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        torch.cuda.synchronize()
        return results


def _leaf(t):
    return t.detach().clone().requires_grad_()


def _fwd_bwd(layer, x, gy):
    """(layer(x), the input gradient of layer's own backward for the output gradient gy)."""
    with torch.no_grad():
        y = layer(x)
    return y, layer._backward(gy, x.shape)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("M", [8, 512])
def test_column_layer_backward_through_collectives(monkeypatch, world, M):
    """Every rank runs the column layer's own forward and backward: gathered output, local output and sequence
    parallelism.  x.grad holds the same bits on every rank and in the first two modes; under sequence parallelism rank
    r's gradient is rows [r M/w, (r+1) M/w) of it; all within the float64 bound of the unsharded input gradient."""
    from bitsandbytes_b200.parallel import ColumnParallelLinear4bit, slice_quantized_weight

    dtype, N, K = torch.bfloat16, 1024, 768
    qW, qs, W64 = _model(N, K, dtype, False, seed=world * M)
    g = torch.Generator().manual_seed(M)
    x = torch.randn(M, K, generator=g).to(dtype).cuda()
    gy = torch.randn(M, N, generator=g).to(dtype).cuda()
    sim = _SimWorld(world, monkeypatch)
    Ms, rows = M // world, N // world

    def step(r, gather_output, sp):
        layer = ColumnParallelLinear4bit(slice_quantized_weight(qW, qs, world, r), N, gather_output=gather_output,
                                         sequence_parallel=sp)
        return _fwd_bwd(layer, x[r * Ms:(r + 1) * Ms] if sp else x,
                        gy if gather_output else gy[:, r * rows:(r + 1) * rows].contiguous())

    gathered = sim.run(lambda r: step(r, True, False))
    local = sim.run(lambda r: step(r, False, False))
    sp = sim.run(lambda r: step(r, False, True))
    nat.check()
    want = gathered[0][1]
    for r in range(world):
        assert torch.equal(gathered[r][1], want) and torch.equal(local[r][1], want), f"rank {r}"
        assert torch.equal(sp[r][1], want[r * Ms:(r + 1) * Ms]), f"SP rank {r}"
        assert torch.equal(sp[r][0], local[r][0]), f"SP forward rank {r}"
    assert_close_to_exact(want, (gy.double() @ W64).cpu().numpy(), "bf16", N)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("M", [8, 512])
def test_row_layer_backward_through_collectives(monkeypatch, world, M):
    """Every rank runs the row layer's own forward and backward.  input_is_parallel: rank r's x_r.grad is its columns
    of the unsharded input gradient; the whole replicated input (input_is_parallel=False): every rank's x.grad is the
    whole input gradient, the ranks' columns in rank order; sequence parallelism: the same as the first, from the
    token rows of the output gradient."""
    from bitsandbytes_b200.parallel import RowParallelLinear4bit, slice_quantized_weight_k

    dtype, N, K = torch.bfloat16, 768, 2048
    qW, qs, W64 = _model(N, K, dtype, True, seed=world + M)
    g = torch.Generator().manual_seed(M + 7)
    x = torch.randn(M, K, generator=g).to(dtype).cuda()
    gy = torch.randn(M, N, generator=g).to(dtype).cuda()
    sim = _SimWorld(world, monkeypatch)
    Ms, kr = M // world, K // world

    def step(r, parallel_input, sp):
        layer = RowParallelLinear4bit(slice_quantized_weight_k(qW, qs, world, r), K, input_is_parallel=parallel_input,
                                      sequence_parallel=sp)
        return _fwd_bwd(layer, x[:, r * kr:(r + 1) * kr] if parallel_input else x, gy[r * Ms:(r + 1) * Ms] if sp else gy)

    sliced = sim.run(lambda r: step(r, True, False))
    whole = sim.run(lambda r: step(r, False, False))
    sp = sim.run(lambda r: step(r, True, True))
    nat.check()
    want = torch.cat([sliced[r][1] for r in range(world)], dim=1)
    for r in range(world):
        assert torch.equal(whole[r][1], want), f"rank {r}"
        assert torch.equal(sp[r][1], sliced[r][1]), f"SP rank {r}"
        assert torch.equal(sp[r][0], sliced[r][0][r * Ms:(r + 1) * Ms]), f"SP forward rank {r}"
    assert_close_to_exact(want, (gy.double() @ W64).cpu().numpy(), "bf16", N)


@pytest.mark.parametrize("loss", ["sum", "mean0", "transposed"])
def test_backward_takes_the_gradient_layouts_autograd_produces(monkeypatch, loss):
    """`.sum()` hands the layers an expanded gradient (strides 0, 0), `.mean(0)` one with strides (0, 1), a transposed
    use a column-major one.  Through autograd at world 1, and through ``_backward`` with the gradient autograd gives the
    output at world 2: x.grad equals the gradient of the same loss passed in contiguous, for both layers."""
    from bitsandbytes_b200.parallel import (ColumnParallelLinear4bit, RowParallelLinear4bit, slice_quantized_weight,
                                            slice_quantized_weight_k)

    dtype, N, K, M = torch.bfloat16, 512, 384, 64
    qW, qs, _ = _model(N, K, dtype, False, seed=31)
    x = torch.randn(M, K, generator=torch.Generator().manual_seed(32)).to(dtype).cuda()
    v = torch.randn(M, generator=torch.Generator().manual_seed(33)).to(dtype).cuda()
    f = {"sum": lambda y: y.sum(), "mean0": lambda y: y.mean(0).sum(),
         "transposed": lambda y: (y.t() @ v).float().sum()}[loss]

    def layers(world, r):
        return (ColumnParallelLinear4bit(slice_quantized_weight(qW, qs, world, r), N),
                RowParallelLinear4bit(slice_quantized_weight_k(qW, qs, world, r), K, input_is_parallel=False))

    for layer in layers(1, 0):
        a, b = _leaf(x), _leaf(x)
        f(layer(a)).backward()
        yd = layer(b).detach().requires_grad_()
        gy, = torch.autograd.grad(f(yd), yd)
        layer(b).backward(gy.contiguous())
        assert torch.equal(a.grad, b.grad)

    def step(r):
        out = []
        for layer in layers(2, r):
            with torch.no_grad():
                y = layer(x)
            yd = y.requires_grad_()
            gy, = torch.autograd.grad(f(yd), yd)
            out.append((layer._backward(gy, x.shape), layer._backward(gy.contiguous(), x.shape)))
        return out

    for res in _SimWorld(2, monkeypatch).run(step):
        for got, want in res:
            assert torch.equal(got, want)
