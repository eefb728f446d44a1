"""GPU tests of the backward of the symmetric-memory routes on one H100: ``reduce_partials_ptrs`` against
``reduce_partials`` on the stacked partials, bit for bit, and its return codes; then, in one process per GPU with real
symmetric memory, every fused route's input gradient against the NCCL route's, a LoRA adapter trained in front of a
fused column -> row pair with ``AdamW8bit``, and that training step captured in a CUDA graph and replayed."""
import ctypes as ct
import os
import subprocess
import sys

import pytest
import torch

from tests import _native as nat

pytestmark = pytest.mark.gpu

_DT = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _partials(n, M, N, seed):
    """n separate [M, N] fp32 partials whose rank-order sum rounds differently from other orders: wide magnitudes."""
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(M, N, generator=g) * 2.0 ** torch.randint(-12, 12, (M, N), generator=g)).cuda()
            for _ in range(n)]


# (M, N): vector-aligned, odd M and N one past / before the vector width of every dtype, one row
_SHAPES = [(64, 1024), (33, 129), (7, 8), (5, 7), (3, 4), (9, 17), (1, 2056)]


@pytest.mark.parametrize("n", range(1, 9))
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("M,N", _SHAPES)
def test_pointer_list_equals_the_stacked_reduction(n, dtype, with_bias, M, N):
    """Separate buffers (tensors, then raw addresses) reduced over all rows and over a row window, into a contiguous
    output and a strided one: the rows of reduce_partials on the stacked partials, bit for bit, nothing written
    outside the window's [rows, N]."""
    from bitsandbytes_b200.backends.cuda import reduce_partials, reduce_partials_ptrs

    td = _DT[dtype]
    parts = _partials(n, M, N, seed=n * 100 + M)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(N)).to(td).cuda() if with_bias else None
    want = reduce_partials(torch.stack(parts), td, bias)
    assert torch.equal(_bits(reduce_partials_ptrs(parts, M, N, td, bias=bias)), _bits(want))
    windows = [(0, M), (M // 3, M - M // 3 - M // 4), (M - 1, 1), (M // 2, 0)]
    for row0, rows in windows:
        for pad in (0, 8, 3):  # row stride N (vector), N + 8 (vector), N + 3 (element by element)
            buf = torch.full((rows + 1, N + pad), float("nan"), device="cuda").to(td)
            out = buf[:rows, :N]
            got = reduce_partials_ptrs([p.data_ptr() for p in parts] if pad else parts, M, N, td, row0, rows, bias,
                                       out=out)
            torch.cuda.synchronize()
            nat.check()
            assert got.data_ptr() == out.data_ptr()
            assert torch.equal(_bits(out), _bits(want[row0:row0 + rows])), (row0, rows, pad)
            assert torch.isnan(buf[rows]).all() and torch.isnan(buf[:, N:]).all()


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_unaligned_partials_take_the_element_path(dtype):
    """Partials 4 bytes off a 16-byte boundary (the vector loads do not apply) give the same bits."""
    from bitsandbytes_b200.backends.cuda import reduce_partials, reduce_partials_ptrs

    td = _DT[dtype]
    M, N = 16, 256
    parts = _partials(3, M, N, seed=5)
    shifted = []
    for p in parts:
        base = torch.empty(M * N + 1, device="cuda")
        base[1:].copy_(p.view(-1))
        shifted.append(base[1:].view(M, N))
    assert shifted[0].data_ptr() % 16 == 4
    want = reduce_partials(torch.stack(parts), td)
    assert torch.equal(_bits(reduce_partials_ptrs(shifted, M, N, td, 4, 8)), _bits(want[4:12]))


def _raw(ptrs, n_parts, row0, rows, out_ptr, bias_ptr, M, N, ldc, dtype_id):
    arr = (ct.c_void_p * max(1, len(ptrs)))(*ptrs)
    rc = nat.lib.cbnb_b200_reduce_partials_ptrs(ct.cast(arr, ct.c_void_p), n_parts, row0, rows, out_ptr, bias_ptr, M,
                                                N, ldc, dtype_id, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


def test_return_codes_write_nothing():
    """Each argument check returns 1 with the error message set, an unknown dtype 100, and nothing is written; the
    Python wrapper refuses the same calls before the library."""
    from bitsandbytes_b200.backends.cuda import reduce_partials_ptrs

    M, N = 16, 64
    parts = _partials(8, M, N, seed=9)
    ptrs = [p.data_ptr() for p in parts]
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float16)
    bias = torch.zeros(N + 1, device="cuda", dtype=torch.float16)
    good = dict(ptrs=ptrs[:4], n_parts=4, row0=0, rows=M, out_ptr=out.data_ptr(), bias_ptr=None, M=M, N=N, ldc=N,
                dtype_id=1)
    bad = [dict(n_parts=0), dict(ptrs=ptrs + ptrs[:1], n_parts=9),       # n_parts outside 1..8
           dict(ptrs=[0, ptrs[1]], n_parts=2),                            # a null partial
           dict(ptrs=[ptrs[0] + 2, ptrs[1]], n_parts=2),                  # a partial off its 4-byte alignment
           dict(out_ptr=out.data_ptr() + 1),                              # out off its element alignment
           dict(bias_ptr=bias.data_ptr() + 1),                            # bias off its element alignment
           dict(row0=-1), dict(rows=-1), dict(row0=1), dict(row0=M, rows=1), dict(rows=M + 1),  # windows past M
           dict(ldc=N - 1)]                                               # ldc < N
    for kw in bad:
        assert _raw(**dict(good, **kw)) == 1, kw
        with pytest.raises(RuntimeError, match="reduce_partials_ptrs"):
            nat.check()
        assert torch.isnan(out).all(), kw
    for dtype_id in (-1, 4, 7):
        assert _raw(**dict(good, dtype_id=dtype_id)) == 100
        nat.check()
        assert torch.isnan(out).all()
    assert _raw(**dict(good, rows=0)) == 0 and torch.isnan(out).all()   # an empty window: nothing to do
    assert _raw(**good) == 0
    nat.check()
    assert torch.isfinite(out).all()
    for kw in [dict(ptrs=[]), dict(ptrs=parts + parts[:1]), dict(row0=M - 1, rows=2), dict(dtype=torch.int32),
               dict(ptrs=[p.half() for p in parts[:2]]), dict(ptrs=[torch.zeros(M * N - 1, device="cuda")]),
               dict(bias=torch.zeros(N, device="cuda")), dict(out=torch.empty(M, N + 1, device="cuda").half())]:
        args = dict(dict(ptrs=parts[:2], M=M, N=N, dtype=torch.float16), **kw)
        with pytest.raises((RuntimeError, ValueError)):
            reduce_partials_ptrs(**args)


# ------------------------------------------------------------------------------------------ processes
_SCRIPT = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["BNB_REPO_ROOT"])
import bitsandbytes_b200 as bnb
import bitsandbytes_b200.functional as F
import bitsandbytes_b200.parallel as par
from bitsandbytes_b200.parallel import (ColumnParallelLinear4bit, ColumnParallelLinear8bitLt, PeerGather, PeerInputGrad,
                                        PeerInt8Input, PeerPartials, RowParallelLinear4bit, RowParallelLinear8bitLt)

rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); mode = os.environ["MODE"]
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
dt = torch.bfloat16
H, I = 1024, 2048


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def same(a, b, what):
    assert a.shape == b.shape and torch.equal(bits(a), bits(b)), f"rank {rank}: {what}"


def weights4(N, K, seed, nested):
    torch.manual_seed(seed)
    return F.quantize_4bit((torch.randn(N, K, device=dev) / K**0.5).to(dt), quant_type="nf4",
                           compress_statistics=nested)


def weights8(N, K, seed):
    torch.manual_seed(seed)
    CB, SCB, _ = F.int8_vectorwise_quant((torch.randn(N, K, device=dev) / K**0.5).half())
    return CB, SCB


def grads(route, layer, x, gy, *peer_args):
    # (fused output, fused x.grad, NCCL output, NCCL x.grad) for the same x and output gradient
    xa = x.detach().clone().requires_grad_()
    ya = route(layer, xa, *peer_args)
    ya.backward(gy)
    xb = x.detach().clone().requires_grad_()
    yb = layer(xb)
    yb.backward(gy)
    return ya, xa.grad, yb, xb.grad


def check_routes(kind, M, threshold):
    torch.manual_seed(100 + M)
    Ms = M // world
    x_full = torch.randn(M, H, device=dev, dtype=dt)
    x_mine = x_full[rank * Ms:(rank + 1) * Ms].contiguous()
    if kind == "4bit":
        up_q, up_s = weights4(I, H, 1, False)
        dn_q, dn_s = weights4(H, I, 2, True)
        col = ColumnParallelLinear4bit.from_quantized(up_q, up_s)
        col_sp = ColumnParallelLinear4bit.from_quantized(up_q, up_s, gather_output=False, sequence_parallel=True)
        row = RowParallelLinear4bit.from_quantized(dn_q, dn_s)
        row_full = RowParallelLinear4bit.from_quantized(dn_q, dn_s, input_is_parallel=False)
        row_sp = RowParallelLinear4bit.from_quantized(dn_q, dn_s, sequence_parallel=True)
        f_col, f_col_sp, f_row, f_row_sp = (par.fused_forward, par.fused_forward_col_sp, par.fused_forward_row,
                                            par.fused_forward_row_sp)
        col_peers, col_sp_peers = PeerGather(M, I, dt, dev), PeerGather(M, H, dt, dev)
        row_peers, row_sp_peers = PeerPartials(M, H, dev), PeerPartials(Ms, H, dev)
    else:
        up_CB, up_SCB = weights8(I, H, 3)
        dn_CB, dn_SCB = weights8(H, I, 4)
        col = ColumnParallelLinear8bitLt.from_quantized(up_CB, up_SCB, threshold=threshold)
        col_sp = ColumnParallelLinear8bitLt.from_quantized(up_CB, up_SCB, threshold=threshold, gather_output=False,
                                                           sequence_parallel=True)
        row = RowParallelLinear8bitLt.from_quantized(dn_CB, dn_SCB, threshold=threshold)
        row_full = RowParallelLinear8bitLt.from_quantized(dn_CB, dn_SCB, threshold=threshold, input_is_parallel=False)
        row_sp = RowParallelLinear8bitLt.from_quantized(dn_CB, dn_SCB, threshold=threshold, sequence_parallel=True)
        f_col, f_col_sp, f_row, f_row_sp = (par.fused_forward_col8, par.fused_forward_col8_sp, par.fused_forward_row8,
                                            par.fused_forward_row8_sp)
        col_peers, col_sp_peers = PeerGather(M, I, dt, dev), PeerInt8Input(M, H, dev)
        row_peers = PeerPartials(M, H, dev, dtype=torch.int32)
        row_sp_peers = PeerPartials(Ms, H, dev, dtype=torch.int32)
    g_col = PeerInputGrad(M, H, torch.float32, dev)
    g_row_full = PeerInputGrad(M, I, dt, dev)
    g_row_sp = PeerInputGrad(M, H, dt, dev)
    h_full = torch.randn(M, I, device=dev, dtype=dt)
    h_mine = h_full[:, rank * I // world:(rank + 1) * I // world].contiguous()
    for step in range(3):  # both slots of every PeerInputGrad, then the first again
        gy = torch.randn(M, I, device=dev, dtype=dt)
        ya, ga, yb, gb = grads(f_col, col, x_full, gy, col_peers, g_col)
        same(ya, yb, f"{kind} column output"); same(ga, gb, f"{kind} column x.grad")
        if world == 1 and kind == "4bit":
            # T(P_0) of the fp32 partial; MatMul4Bit.backward rounds cuBLAS's own bf16 output, which may take another
            # kernel: the same up to that rounding, and reported when the bits differ
            same(ga, par.input_grad_dequant_matmul(gy, col.shard, torch.float32).to(dt), "4bit column T(P_0)")
            xc = x_full.detach().clone().requires_grad_()
            bnb.matmul_4bit(xc, up_q.t(), up_s).backward(gy)
            torch.testing.assert_close(ga, xc.grad, rtol=1.6e-2, atol=1e-3)
            if not torch.equal(bits(ga), bits(xc.grad)):
                print(f"M={M}: column x.grad differs from MatMul4Bit.backward in the last bits")
        gy = torch.randn(M, I // world, device=dev, dtype=dt)
        ya, ga, yb, gb = grads(f_col_sp, col_sp, x_mine, gy, col_sp_peers, g_col)
        same(ya, yb, f"{kind} SP column output"); same(ga, gb, f"{kind} SP column x.grad")
        gy = torch.randn(M, H, device=dev, dtype=dt)
        ya, ga, yb, gb = grads(f_row, row, h_mine, gy, row_peers, g_row_full)
        same(ya, yb, f"{kind} row output"); same(ga, gb, f"{kind} row x.grad")
        if world == 1 and kind == "4bit":
            xc = h_mine.detach().clone().requires_grad_()
            bnb.matmul_4bit(xc, dn_q.t(), dn_s).backward(gy)
            same(ga, xc.grad, "4bit row x.grad against MatMul4Bit.backward")
        ya, ga, yb, gb = grads(f_row, row_full, h_full, gy, row_peers, g_row_full)
        same(ya, yb, f"{kind} row (whole input) output"); same(ga, gb, f"{kind} row (whole input) x.grad")
        gy = torch.randn(Ms, H, device=dev, dtype=dt)
        ya, ga, yb, gb = grads(f_row_sp, row_sp, h_mine, gy, row_sp_peers, g_row_sp)
        same(ya, yb, f"{kind} SP row output"); same(ga, gb, f"{kind} SP row x.grad")
    torch.cuda.synchronize()


def check_shared_output_slots(kind, M):
    # three gathered column calls through one PeerGather (the slot of the first is rewritten by the third) before one
    # backward, each output saved by SiLU: the NCCL route's outputs and gradients
    torch.manual_seed(200 + M)
    if kind == "4bit":
        q, st = weights4(I, H, 10, False)
        col, route = ColumnParallelLinear4bit.from_quantized(q, st), par.fused_forward
    else:
        CB, SCB = weights8(I, H, 11)
        col, route = ColumnParallelLinear8bitLt.from_quantized(CB, SCB), par.fused_forward_col8
    peers, g = PeerGather(M, I, dt, dev), PeerInputGrad(M, H, torch.float32, dev)
    xs = [torch.randn(M, H, device=dev, dtype=dt) for _ in range(3)]
    gys = [torch.randn(M, I, device=dev, dtype=dt) for _ in range(3)]

    def run(fn):
        xa = [x.clone().requires_grad_() for x in xs]
        ys = [torch.nn.functional.silu(fn(x)) for x in xa]
        sum((y.float() * gy.float()).sum() for y, gy in zip(ys, gys)).backward()
        return [y.detach() for y in ys], [x.grad for x in xa]

    (yf, gf), (yn, gn) = run(lambda x: route(col, x, peers, g)), run(col)
    for i in range(3):
        same(yf[i], yn[i], f"{kind}: call {i} output through a shared PeerGather")
        same(gf[i], gn[i], f"{kind}: call {i} x.grad through a shared PeerGather")


class Model(torch.nn.Module):
    # x -> LoRA adapter -> column layer -> SiLU -> row layer, through the fused routes or the layers' own forward
    def __init__(self, kind, M, fused, seed=7):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.A = torch.nn.Parameter((torch.randn(16, H, generator=g) / H**0.5).to(dt).to(dev))
        self.B = torch.nn.Parameter((torch.randn(H, 16, generator=g) * 0.01).to(dt).to(dev))
        self.fused, self.kind = fused, kind
        if kind == "4bit":
            up_q, up_s = weights4(I, H, 5, False)
            dn_q, dn_s = weights4(H, I, 6, True)
            self.col = ColumnParallelLinear4bit.from_quantized(up_q, up_s, gather_output=fused)
            self.row = RowParallelLinear4bit.from_quantized(dn_q, dn_s, input_is_parallel=not fused)
            self.f_col, self.f_row = par.fused_forward, par.fused_forward_row
        else:
            up_CB, up_SCB = weights8(I, H, 8)
            dn_CB, dn_SCB = weights8(H, I, 9)
            self.col = ColumnParallelLinear8bitLt.from_quantized(up_CB, up_SCB, gather_output=fused)
            self.row = RowParallelLinear8bitLt.from_quantized(dn_CB, dn_SCB, input_is_parallel=not fused)
            self.f_col, self.f_row = par.fused_forward_col8, par.fused_forward_row8
        if fused:
            # the gathered output of the fused column route, of which the row layer (whole input) takes its columns
            self.col_peers, self.row_peers = PeerGather(M, I, dt, dev), PeerPartials(
                M, H, dev, dtype=torch.float32 if kind == "4bit" else torch.int32)
            self.g_col, self.g_row = PeerInputGrad(M, H, torch.float32, dev), PeerInputGrad(M, I, dt, dev)

    def forward(self, x):
        x = x + (x @ self.A.t()) @ self.B.t()
        if self.fused:
            h = torch.nn.functional.silu(self.f_col(self.col, x, self.col_peers, grad_peers=self.g_col))
            return self.f_row(self.row, h, self.row_peers, grad_peers=self.g_row)
        h = torch.nn.functional.silu(self.col(x))
        if world > 1:
            raise RuntimeError("the reference pair is the one-rank layers")
        return self.row(h)


def train(kind, M, steps=3):
    torch.manual_seed(11)
    data = [(torch.randn(M, H, device=dev, dtype=dt), torch.randn(M, H, device=dev, dtype=dt)) for _ in range(steps)]
    models = [Model(kind, M, fused) for fused in (True, False)] if world == 1 else [Model(kind, M, True)]
    opts = [bnb.optim.AdamW8bit([m.A, m.B], lr=1e-3) for m in models]
    for x, y in data:
        for m, o in zip(models, opts):
            o.zero_grad(set_to_none=True)
            torch.nn.functional.mse_loss(m(x).float(), y.float()).backward()
            o.step()
    torch.cuda.synchronize()
    assert not torch.equal(models[0].B, Model(kind, M, False).B), "the adapter did not train"
    if world == 1:
        for a, b in ((models[0].A, models[1].A), (models[0].B, models[1].B)):
            same(a, b, f"{kind}: the adapter trained through the fused routes")


def graph(kind, M):
    # the fused training step captured once and replayed: the bits of the same step run eagerly
    torch.manual_seed(12)
    data = [(torch.randn(M, H, device=dev, dtype=dt), torch.randn(M, H, device=dev, dtype=dt)) for _ in range(6)]
    ma, mb = Model(kind, M, True), Model(kind, M, True)
    oa = bnb.optim.AdamW8bit([ma.A, ma.B], lr=1e-3, capturable=True)
    ob = bnb.optim.AdamW8bit([mb.A, mb.B], lr=1e-3, capturable=True)

    def step(m, o, x, y):
        loss = torch.nn.functional.mse_loss(m(x).float(), y.float())
        loss.backward()
        o.step()
        return loss

    sx, sy = data[0][0].clone(), data[0][1].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for x, y in data[:2]:
            oa.zero_grad(set_to_none=True); ob.zero_grad(set_to_none=True)
            sx.copy_(x); sy.copy_(y)
            step(ma, oa, sx, sy); step(mb, ob, x, y)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    oa.zero_grad(set_to_none=True)
    with torch.cuda.graph(g):
        sloss = step(ma, oa, sx, sy)
    for x, y in data[2:]:
        sx.copy_(x); sy.copy_(y)
        g.replay()
        ob.zero_grad(set_to_none=True)
        want = step(mb, ob, x, y)
        torch.cuda.synchronize()
        same(sloss.detach(), want.detach(), f"{kind}: replayed loss")
        same(ma.A, mb.A, f"{kind}: replayed A"); same(ma.B, mb.B, f"{kind}: replayed B")


if mode == "routes":
    for kind in ("4bit", "int8"):
        for M in (64, 256):
            for threshold in ((0.0,) if kind == "4bit" else (0.0, 6.0)):
                check_routes(kind, M, threshold)
            check_shared_output_slots(kind, M)
elif mode == "train":
    for kind in ("4bit", "int8"):
        train(kind, 128)
elif mode == "graph":
    for kind in ("4bit", "int8"):
        graph(kind, 128)
dist.barrier()
dist.destroy_process_group()
print("FUSED_BWD_OK", rank)
"""


def _run(tmp_path, nproc, mode):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "fused_bwd.py"
    script.write_text(_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNB_REPO_ROOT=root, MODE=mode)
    port = 29611 + 4 * nproc + ["routes", "train", "graph"].index(mode)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and r.stdout.count("FUSED_BWD_OK") == nproc, r.stdout[-3000:] + r.stderr[-4000:]


@pytest.mark.parametrize("nproc", [1, 2])
def test_processes_fused_gradients_equal_nccl(tmp_path, nproc):
    """One process per GPU, real symmetric memory: each of the eight fused routes gives the output and x.grad of the
    same layer's NCCL route, bit for bit, on every rank (and, for the 4-bit layers at one rank, MatMul4Bit.backward's
    gradient), also with three gathered column calls sharing one PeerGather before one backward.  One process runs
    the symmetric-memory code at a world of 1, where the row routes exchange nothing and the column routes reduce one
    slot; the copies into the peers' slots run on real symmetric memory only with two GPUs."""
    _run(tmp_path, nproc, "routes")


@pytest.mark.parametrize("nproc", [1, 2])
def test_processes_lora_trains_through_fused_routes(tmp_path, nproc):
    """A LoRA adapter in front of a fused column -> row pair, mse loss and AdamW8bit over three steps: at one rank the
    adapter ends bit-identical to the same steps through the layers' own forward; at two, it trains."""
    _run(tmp_path, nproc, "train")


def test_process_fused_training_step_replays_in_a_cuda_graph(tmp_path):
    """The fused training step (4-bit layers, and int8 at threshold 0) captured once and replayed four times: the loss
    and the adapter equal the same steps run eagerly, bit for bit."""
    _run(tmp_path, 1, "graph")
