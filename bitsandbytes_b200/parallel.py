"""Column- and row-sharded Linear4bit: one process per GPU, ``torch.distributed`` (NCCL over NVLink 5 /
NVSwitch) for the plumbing.  New functionality -- the reference is a single-device library
(SURVEY.md section 2.3); what it does provide is proof that byte-range sharding of a packed
4-bit weight is lossless (reference tests/test_linear4bit.py:256-283).

Sharding rule (SURVEY.md section 8e).  ``W[N, K]`` is packed row-major, quantisation blocks
run along K and never straddle rows when ``K % blocksize == 0``, so a row range
``[n0, n1)`` owns the contiguous byte range ``[n0*K/2, n1*K/2)`` and the contiguous
absmax range ``[n0*K/bs, n1*K/bs)``.  With double quantisation the 8-bit absmax codes are
sliced the same way and the level-2 statistics (one fp32 per 256 blocks), the level-2 code
book and the offset are addressed through the shard's first *global* block index, which must
be a multiple of 256 so that ``global_block >> 8`` stays aligned: rows per shard * K / bs %
256 == 0.  The weight is quantised ONCE globally and then sliced, never re-quantised per
shard, so every shard reproduces the single-GPU result bit for bit.

Forward: every rank holds the replicated activations ``x[M, K]``, computes its
``[M, N/world]`` slice with the fused kernel *directly into its columns of the full-width
output* (strided-output entry point of the C ABI) and the slices are exchanged with one
all-gather.  The gather is along the inner dimension of a row-major matrix, which
``all_gather_into_tensor`` cannot write in place, so the exchange runs on a ``[world, M,
N/world]`` staging buffer; ``gather_output=False`` hands back the local slice instead (what
a following row-parallel layer wants).

Fused exchange (``PeerGather`` + ``fused_forward``): the output lives in symmetric memory
(``torch.distributed._symmetric_memory``: one ``[M, N]`` buffer per rank, every rank holds the
peers' mappings) and the GEMM epilogue stores each output element into ITS columns of EVERY rank's
buffer -- the all-gather rides on the kernel's own stores over NVLink / NVSwitch, tile by tile,
there is no separate collective and no permute; one symmetric-memory barrier per step publishes
the result.  Buffers alternate between two slots so that a rank may start step i + 1 while a peer
still reads step i.

Row sharding (``RowParallelLinear4bit``, the layer after a column-parallel one with
``gather_output=False``: o_proj, down_proj).  Rank r owns the input features ``[r*K/w, (r+1)*K/w)``:
``W[:, k0:k1]``, strided in the packed layout, is repacked once at load by
``slice_quantized_weight_k`` (``K % (world * blocksize) == 0`` and ``(K/world) % 64 == 0``, which keeps
the shard on the tensor-core kernels).  Double-quantised statistics do not survive a column cut (a
level-2 group of 256 blocks straddles shards), so the shard's scales become plain fp32 absmax, computed
as the kernels fetch them (``code2[a8] * absmax2`` rounded, ``+ offset`` rounded): the shard decodes to
the same weights bit for bit.  Rank r computes the fp32 partial ``P_r = x_r . dequant(W_r)^T`` with no
bias and no rounding (``gemm_4bit_partial``), every rank gathers all of them, and every rank produces
``y = T((((P_0 + P_1) + P_2) + ... + P_{w-1}) + bias)``: an fp32 sum in rank order, the bias added in
fp32, one rounding (``reduce_partials``).  Every rank holds the same bits, the fused and the NCCL
exchange give the same bits, and the result differs from the unsharded layer only by the order of the
fp32 sum, as split-K does; with one rank it is the unsharded result exactly.  The exchange moves
``4 * M * N * world`` bytes per rank.  Unfused, the partials meet in a ``[world, M, N]`` fp32 stage
through ``all_gather_into_tensor``; fused (``PeerPartials`` + ``fused_forward_row``), the GEMM epilogue
stores ``P_r`` into slot r of every rank's symmetric ``[world, M, N]`` buffer, one barrier publishes
them and each rank reduces locally.

Sequence parallelism (``sequence_parallel=True`` on both layers, Megatron's ``[s, b, h]`` layout).  The activations
between the column -> row pair (norms, residuals) are sharded by token: the first dimension of the activation is split
over the ranks, so the flattened rows ``[r*M/w, (r+1)*M/w)`` belong to rank r, and ``x.shape[0] % world == 0`` is
required (``ValueError`` otherwise).  The column layer takes its rank's ``[M/w, ..., K]`` tokens, all-gathers them
along dim 0 (NCCL ``all_gather_into_tensor``, or ``fused_forward_col_sp``: a copy into this rank's rows of every
rank's symmetric ``[M, K]`` buffer and one barrier) and returns its ``[M, ..., N/w]`` features, bit for bit the
non-SP layer on the gathered input (it needs ``gather_output=False``).  The row layer runs the same partial GEMM as
without SP (same M: same kernel, tile and K split) and hands back only its tokens, ``[x.shape[0]/w, ..., N]``, bit for
bit rows ``[r*M/w, (r+1)*M/w)`` of the non-SP output, since ``reduce_partials`` works element by element in rank order.
Unfused, the ``[M, N]`` partial is exchanged by ``all_to_all_single`` into a ``[w, M/w, N]`` buffer (not NCCL's
reduce-scatter, whose summation order is not rank order); fused (``fused_forward_row_sp``, ``PeerPartials(M/w, N)``),
the GEMM epilogue stores the rows of rank s into slot r of rank s's buffer (``gemm_4bit_partial_scatter``).  Either way
a rank sends ``4*M*N*(w-1)/w`` bytes, w times less than the all-gather of the partials, and reduces ``4*M*N`` bytes
instead of ``4*w*M*N``.

Training (QLoRA under tensor and sequence parallelism).  Both layers' forward runs through a ``torch.autograd.Function``
(the same bits as before) whose backward gives the input gradient ``grad_x = grad_y . dequant(W)`` and nothing else:
the sharded weights and biases stay frozen.  The column layer's rank r holds ``P_r = G_r . dequant(W_r)`` in fp32, ``G_r``
its columns of ``grad_y``, and the partials meet as in the row layer's forward: all-gathered and summed in rank order by
``reduce_partials`` (every rank holds the same bits; with one rank ``grad_x = T(P_0)``), or, with sequence parallelism,
exchanged by token with ``all_to_all_single`` so that each rank reduces only its tokens' rows, which are the non-SP
result's rows bit for bit.  The row layer needs no exchange, ``grad_x_r = grad_y . dequant(W_r)`` rounded once, after an
all-gather of ``grad_y``'s token rows under sequence parallelism; with ``input_is_parallel=False`` (the whole replicated
input, of which the layer uses its columns) the ranks' ``grad_x_r`` are all-gathered along the features, in rank order,
into the whole input gradient.  Both products run as dequantise + cuBLAS (:func:`input_grad_dequant_matmul`, chosen in
``_input_grad`` from timings against a fused 4-bit input-gradient kernel, DESIGN.md section 6).  The tensor-parallel
LLM.int8() layers below share this backward (``_ColumnInputGrad``, ``_RowInputGrad``); only the dequantised weight
differs (``Shard4bit.dequantize``, ``Shard8bit.dequantize``).

The ``fused_forward*`` routes train when given ``grad_peers`` (:class:`PeerInputGrad`, two symmetric-memory slots): the
forward and the backward are the layer's, through the same ``torch.autograd.Function``, each with its exchange through
symmetric memory instead of NCCL.  The column layer's rank r stores its fp32 partial into its own slot,
one barrier, and each rank reduces the peers' slots in rank order (``reduce_partials_ptrs``, the arithmetic of
``reduce_partials``): all M rows, or only its tokens' rows under sequence parallelism.  The row layer copies its
tokens' rows of ``grad_y`` (sequence parallelism) or its columns of the input gradient (``input_is_parallel=False``)
into every rank's slot, one barrier.  The gradients are the NCCL route's bit for bit.  Without ``grad_peers`` the fused
routes refuse an input that requires grad, as before.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
import torch.distributed as dist

from . import functional as F
from .backends.cuda import (gemm_4bit_grouped_into, gemm_4bit_grouped_partial, gemm_4bit_into, gemm_4bit_multi_out,
                            gemm_4bit_partial, gemm_4bit_partial_scatter, int8_dequant_rows, int8_gemm_multi_out,
                            int8_gemm_partial_scatter, int8_outlier_operands, int8_quant_with_stats,
                            int8_reduce_partials, int8_row_stats, int8_vectorwise_quant_flags, int8_zero_columns,
                            reduce_partials, reduce_partials_grouped, reduce_partials_ptrs)


@dataclass
class Shard4bit:
    """The slice of a quantised [N, K] weight owned by one rank; with ``experts`` = E > 1, the slice of every expert of
    an [E, N, K] expert tensor, stacked as an [E, rows, K] weight."""

    packed: torch.Tensor            # uint8 [experts*rows*K/2]
    absmax: torch.Tensor            # fp32 [rows*K/bs]  (plain)  |  level-2 absmax slice (nested)
    absmax_8bit: Optional[torch.Tensor]
    absmax_code: Optional[torch.Tensor]
    absmax_offset: Optional[torch.Tensor]
    rows: int
    row0: int
    K: int
    blocksize: int
    quant_type: str
    k0: int = 0                     # first input feature of a K shard (slice_quantized_weight_k)
    experts: int = 1                # experts of a grouped shard (slice_grouped_weight, slice_grouped_weight_k)

    def dequantize(self, dtype: torch.dtype) -> torch.Tensor:
        """The shard's weight ``[experts * rows, K]`` decoded to ``dtype`` as ``dequantize_4bit`` decodes it."""
        scales = self.absmax
        if self.absmax_8bit is not None:
            scales = _nested_scales(self.absmax_8bit, self.absmax, self.absmax_code, self.absmax_offset)
        out = torch.empty((self.experts * self.rows, self.K), device=self.packed.device, dtype=dtype)
        return F.dequantize_4bit(self.packed, absmax=scales, out=out, blocksize=self.blocksize,
                                 quant_type=self.quant_type)


def shard_rows(N: int, world: int, rank: int) -> tuple[int, int]:
    if N % world != 0:
        raise ValueError(f"out_features ({N}) must be divisible by the world size ({world})")
    rows = N // world
    return rank * rows, rows


def slice_quantized_weight(packed: torch.Tensor, qs: F.QuantState, world: int, rank: int) -> Shard4bit:
    """Cut rank's row range out of a globally quantised weight (no re-quantisation)."""
    N, K = qs.shape
    bs = qs.blocksize
    if K % bs != 0:
        raise ValueError(f"in_features ({K}) must be a multiple of the blocksize ({bs}) to shard by rows")
    row0, rows = shard_rows(N, world, rank)
    flat = packed.reshape(-1).view(torch.uint8) if packed.dtype != torch.uint8 else packed.reshape(-1)
    b0, b1 = row0 * K // 2, (row0 + rows) * K // 2
    a0, a1 = row0 * K // bs, (row0 + rows) * K // bs
    if qs.nested:
        if a0 % 256 != 0 or (a1 - a0) % 256 != 0:
            raise ValueError("double-quantised shards must start and end on a 256-block boundary "
                             f"(rows*K/blocksize = {a1 - a0})")
        return Shard4bit(packed=flat[b0:b1].contiguous(), absmax=qs.state2.absmax[a0 // 256:a1 // 256].contiguous(),
                         absmax_8bit=qs.absmax[a0:a1].contiguous(), absmax_code=qs.state2.code,
                         absmax_offset=qs.offset.reshape(1).float(), rows=rows, row0=row0, K=K, blocksize=bs,
                         quant_type=qs.quant_type)
    return Shard4bit(packed=flat[b0:b1].contiguous(), absmax=qs.absmax[a0:a1].contiguous(), absmax_8bit=None,
                     absmax_code=None, absmax_offset=None, rows=rows, row0=row0, K=K, blocksize=bs,
                     quant_type=qs.quant_type)


class _ColumnInputGrad:
    """The backward of a column-parallel layer, shared by the 4-bit and the int8 layers: the layer provides ``shard``
    (``rows``, ``row0``, ``K`` and ``dequantize(dtype)``), ``group`` and ``sequence_parallel``."""

    def input_grad_partial(self, grad_y: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
        """This rank's fp32 partial ``P_r = G_r . W_r`` of the input gradient into ``out`` ``[M, K]``: ``G_r`` is
        ``grad_y`` itself (``[M, rows]``, this rank's output) or, for the ``[M, world * rows]`` gathered output, this
        rank's columns of it, read in place."""
        s = self.shard
        G = grad_y.reshape(-1, grad_y.shape[-1])
        if G.shape[1] != s.rows:
            G = G[:, s.row0:s.row0 + s.rows]
        return _input_grad(G, s, out)

    def _grad_slot(self, x: torch.Tensor, sp: bool):
        """(shape, dtype) of the slot the fused backward exchanges through for the input ``x`` of a route in mode ``sp``:
        fp32 ``[M, K]``, M all tokens (``world`` times this rank's under sequence parallelism)."""
        world = _group_world_rank(self.group)[0] if sp else 1
        return (world * (x.numel() // self.shard.K), self.shard.K), torch.float32

    def _backward(self, grad_y: torch.Tensor, x_shape, peers: Optional["PeerInputGrad"] = None) -> torch.Tensor:
        s = self.shard
        world, rank = _group_world_rank(self.group)
        M = grad_y.numel() // grad_y.shape[-1]
        if peers is not None:
            # the partial into this rank's own slot; once every rank's is complete, each rank reduces, in rank order,
            # the rows it owns (its tokens under sequence parallelism, all M otherwise) straight from the peers' slots
            local, bases, handle = peers.slot()
            self.input_grad_partial(grad_y, local)
            handle.barrier(channel=0)  # every rank's partial is complete
            row0, rows = (rank * (M // world), M // world) if self.sequence_parallel else (0, M)
            return reduce_partials_ptrs(peers.scatter_ptrs(bases, 0), M, s.K, grad_y.dtype, row0, rows).view(x_shape)
        if self.sequence_parallel and world > 1:
            # the partial over all M tokens, its rows sent to the ranks that own them: chunk r of recv is rank r's
            send = torch.empty((world, M // world, s.K), device=grad_y.device)
            self.input_grad_partial(grad_y, send.view(M, s.K))
            recv = torch.empty_like(send)
            dist.all_to_all_single(recv, send, group=self.group)
            return reduce_partials(recv, grad_y.dtype).view(x_shape)
        stage = torch.empty((world, M, s.K), device=grad_y.device)
        self.input_grad_partial(grad_y, stage[rank])
        if world > 1:
            dist.all_gather_into_tensor(stage.view(-1), stage[rank].reshape(-1), group=self.group)
        return reduce_partials(stage, grad_y.dtype).view(x_shape)


class _RowInputGrad:
    """The backward of a row-parallel layer, shared by the 4-bit and the int8 layers: the layer provides ``shard``
    (``rows``, ``K`` and ``dequantize(dtype)``), ``group``, ``input_is_parallel`` and ``sequence_parallel``."""

    def input_grad(self, grad_y: torch.Tensor) -> torch.Tensor:
        """``grad_x_r = grad_y . W_r`` ``[M, K/world]`` for the ``[..., N]`` output gradient of all M tokens."""
        s = self.shard
        G = grad_y.reshape(-1, s.rows)
        return _input_grad(G, s, torch.empty((G.shape[0], s.K), device=G.device, dtype=G.dtype))

    def _grad_slot(self, x: torch.Tensor, sp: bool):
        """(shape, dtype) of the slot the fused backward exchanges through for the input ``x``, or (None, None) when it
        exchanges nothing; it follows the layer's own flags, whatever the route's mode ``sp``.  Sequence parallelism with
        ``input_is_parallel=False`` exchanges twice, ``[M, N]`` then ``[M, in_features]``, which one PeerInputGrad serves
        only when the two agree."""
        world, _ = _group_world_rank(self.group)
        M = x.numel() // x.shape[-1]
        shapes = set()
        if self.sequence_parallel and world > 1:
            shapes.add((M, self.out_features))
        if not self.input_is_parallel and world > 1:
            shapes.add((M, self.in_features))
        if len(shapes) > 1:
            raise ValueError("a sequence-parallel row layer with input_is_parallel=False exchanges [M, out_features] and "
                             "[M, in_features] gradients: one PeerInputGrad serves both only when they are equal")
        return (shapes.pop(), x.dtype) if shapes else (None, None)

    def _backward(self, grad_y: torch.Tensor, x_shape, peers: Optional["PeerInputGrad"] = None) -> torch.Tensor:
        world, rank = _group_world_rank(self.group)
        if self.sequence_parallel and world > 1:
            # this rank's tokens' rows of grad_y -> all M rows, in rank order (= token order)
            if peers is None:
                full = torch.empty((world * grad_y.shape[0], *grad_y.shape[1:]), device=grad_y.device,
                                   dtype=grad_y.dtype)
                dist.all_gather_into_tensor(full, grad_y.contiguous(), group=self.group)
            else:  # copied into this rank's rows of every rank's slot
                Ms, N = grad_y.numel() // grad_y.shape[-1], grad_y.shape[-1]
                full, _, handle = peers.slot()
                for r in range(world):
                    handle.get_buffer(r, (Ms, N), grad_y.dtype, rank * Ms * N).copy_(grad_y.reshape(Ms, N))
                handle.barrier(channel=0)  # every rank's rows have landed everywhere
            grad_y = full
        g = self.input_grad(grad_y)
        if not self.input_is_parallel and world > 1:
            # the layer took the whole (replicated) input and used only its columns: the input gradient is every rank's
            # columns, all-gathered in rank order (the backward of the scatter)
            if peers is None:
                parts = torch.empty((world, *g.shape), device=g.device, dtype=g.dtype)
                dist.all_gather_into_tensor(parts, g, group=self.group)
                g = parts.permute(1, 0, 2).reshape(g.shape[0], world * g.shape[1])
            else:  # copied into this rank's columns of every rank's slot
                M, k0 = g.shape[0], self.shard.k0
                full, _, handle = peers.slot()
                for r in range(world):
                    handle.get_buffer(r, (M, self.in_features), g.dtype, 0)[:, k0:k0 + g.shape[1]].copy_(g)
                handle.barrier(channel=0)  # every rank's columns have landed everywhere
                # a copy: the slot is rewritten two exchanges later, and autograd may keep the gradient (x.grad)
                g = full.clone()
        return g.view(x_shape)


class _ParallelFn(torch.autograd.Function):
    """A tensor-parallel layer's forward (``layer._forward``, exchanging through NCCL, or through ``peers`` in the mode
    ``sp`` of a fused route), with the input gradient as its backward (``layer._backward``, exchanging through NCCL, or
    through ``grad_peers`` for a fused route): the shard and the bias stay frozen.  ``copy_out``: the forward returns a
    copy of its output (see :func:`_fused_route`)."""

    @staticmethod
    def forward(ctx, x, layer, peers=None, sp=None, grad_peers=None, copy_out=False):
        ctx.layer, ctx.x_shape, ctx.peers = layer, x.shape, grad_peers
        y = layer._forward(x, peers, sp)
        return y.clone() if copy_out else y

    @staticmethod
    def backward(ctx, grad_y):
        return ctx.layer._backward(grad_y, ctx.x_shape, ctx.peers), None, None, None, None, None


class ColumnParallelLinear4bit(_ColumnInputGrad, torch.nn.Module):
    """``y = x @ dequant(W)^T + b`` with W's output features split across the process group."""

    def __init__(self, shard: Shard4bit, out_features: int, bias: Optional[torch.Tensor] = None,
                 group: Optional[dist.ProcessGroup] = None, gather_output: bool = True,
                 sequence_parallel: bool = False):
        super().__init__()
        if sequence_parallel and gather_output:
            raise ValueError("sequence_parallel=True hands each rank all tokens of its feature slice: it needs "
                             "gather_output=False")
        self.shard = shard
        self.out_features = out_features
        self.group = group
        self.gather_output = gather_output
        self.sequence_parallel = sequence_parallel
        self.bias_shard = None if bias is None else bias[shard.row0:shard.row0 + shard.rows].contiguous()
        self._stage = None

    @classmethod
    def from_quantized(cls, packed, qs: F.QuantState, bias=None, group=None, gather_output=True,
                       sequence_parallel=False):
        world, rank = _group_world_rank(group)
        return cls(slice_quantized_weight(packed, qs, world, rank), qs.shape[0], bias, group, gather_output,
                   sequence_parallel)

    def local_forward(self, x: torch.Tensor, out: Optional[torch.Tensor] = None, ldc: Optional[int] = None):
        """This rank's [M, rows] slice; written into ``out`` (row stride ``ldc`` elements) if given."""
        s = self.shard
        M = x.numel() // s.K
        if out is None:
            out = torch.empty((M, s.rows), device=x.device, dtype=x.dtype)
            ldc = s.rows
        gemm_4bit_into(x, s.packed, (s.rows, s.K), s.absmax, s.blocksize, s.quant_type, self.bias_shard, s.absmax_8bit,
                       s.absmax_code, s.absmax_offset, out, ldc)
        return out

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _ParallelFn.apply(x, self)

    def _forward(self, x: torch.Tensor, peers: Optional["PeerGather"] = None,
                 sp: Optional[bool] = None) -> torch.Tensor:
        """The layer's output.  ``sp`` (default: ``sequence_parallel``) chooses the mode.  With ``peers`` the exchange
        goes through its symmetric-memory slot, followed by one barrier: under sequence parallelism this rank's tokens
        are copied into its rows of every rank's ``[M, K]`` slot and the local output returned; otherwise the GEMM
        epilogue stores the output into this rank's columns of every rank's ``[M, N]`` slot (the NCCL gather filling
        the slot when the GEMM refuses the call), and the slot itself is returned, whatever ``gather_output`` says."""
        s = self.shard
        world, _ = _group_world_rank(self.group)
        if self.sequence_parallel if sp is None else sp:
            if peers is not None:
                Ms = x.numel() // s.K
                _check_peers(peers, peers.world * Ms, s.K, x.dtype, "token count / input width / dtype")
                local, _, handle = peers.slot()
                xs = x.reshape(Ms, s.K)
                for r in range(peers.world):
                    handle.get_buffer(r, (Ms, s.K), x.dtype, peers.rank * Ms * s.K).copy_(xs)
                handle.barrier(channel=0)  # every rank's tokens have landed everywhere
                return self.local_forward(local).view(peers.world * x.shape[0], *x.shape[1:-1], s.rows)
            if world > 1:
                full = torch.empty((world * x.shape[0], *x.shape[1:]), device=x.device, dtype=x.dtype)
                dist.all_gather_into_tensor(full, x.contiguous(), group=self.group)
                x = full
        lead = x.shape[:-1]
        M = x.numel() // s.K
        if peers is not None:
            _check_peers(peers, M, self.out_features, x.dtype, "output shape / dtype")
            local, bases, handle = peers.slot()
            ptrs = peers.dest_ptrs(bases, s.row0 * local.element_size())
            ok = gemm_4bit_multi_out(x, s.packed, (s.rows, s.K), s.absmax, s.blocksize, s.quant_type, self.bias_shard,
                                     s.absmax_8bit, s.absmax_code, s.absmax_offset, ptrs, peers.N)
            if not ok:  # shape outside the tensor-core kernel: local slice + NCCL all-gather into the same slot
                local.copy_(_gather_columns(self, x, M, x.dtype, x.device))
            handle.barrier(channel=0)  # every rank's stores have landed everywhere
            return local
        if world == 1 or not self.gather_output:
            return self.local_forward(x).view(*lead, s.rows)
        return _gather_columns(self, x, M, x.dtype, x.device).reshape(*lead, world * s.rows)


def input_grad_dequant_matmul(G: torch.Tensor, shard, dtype: torch.dtype) -> torch.Tensor:
    """``G . W`` ``[M, K]`` by dequantise + ``torch.matmul``: the shard's weight (a :class:`Shard4bit` decoded as
    ``dequantize_4bit`` decodes it, a :class:`Shard8bit` as ``MatMul8bitLt.backward`` dequantises it) in G's dtype,
    multiplied by cuBLAS with an output of ``dtype`` -- G's dtype, or fp32 on the fp32 accumulation of the 16-bit
    operands for a partial."""
    W = shard.dequantize(G.dtype)
    if dtype == G.dtype:
        return torch.matmul(G, W)
    if G.dtype != torch.float32:
        return torch.mm(G, W, out_dtype=torch.float32)  # 16-bit operands, fp32 accumulation and output
    return torch.matmul(G.float(), W.float())


def _input_grad(G: torch.Tensor, shard, out: torch.Tensor) -> torch.Tensor:
    """``out[M, K] = G . W`` (``G`` ``[M, rows]`` in any layout, ``shard`` a Shard4bit or Shard8bit): fp32 ``out``
    receives the unrounded partial, one of G's dtype the sum rounded once.  The route is dequantise + cuBLAS -- with an
    fp32 output from the 16-bit operands for a partial -- at every M: on an H100 it was as fast as a fused 4-bit
    input-gradient kernel or faster at every shape and token count measured but one (4096 x 4096 at 256 tokens, not a
    range of M; DESIGN.md section 6), and that kernel was removed.  The int8 layers have no other route."""
    out.copy_(input_grad_dequant_matmul(G, shard, out.dtype))
    return out


def _fused_route(what: str, layer, x: torch.Tensor, peers, sp: bool, grad_peers: Optional["PeerInputGrad"],
                 copy_out: bool = False) -> torch.Tensor:
    """``layer._forward(x, peers, sp)``, a fused route's forward, as it is or, for an input that requires grad, through
    :class:`_ParallelFn` with the layer's backward exchanging through ``grad_peers``, checked once here against the slot
    that backward exchanges through (``layer._grad_slot``).  Without ``grad_peers`` such an input is refused: the route
    would drop its gradient.

    ``copy_out``: the forward returns its symmetric-memory output slot, which the peers' GEMM epilogues rewrite two
    calls later.  Inference uses the output at once; autograd may keep it until the backward (SiLU, a norm or a product
    save their input), so a training call returns a copy."""
    if not (torch.is_grad_enabled() and x.requires_grad):
        return layer._forward(x, peers, sp)
    if grad_peers is None:
        raise RuntimeError(f"{what} is inference only without grad_peers and would drop the input gradient: pass "
                           "grad_peers=PeerInputGrad(...) to train through it, call the layer itself, or run this under "
                           "torch.no_grad()")
    _check_peer_grad(grad_peers, layer.group, *layer._grad_slot(x, sp))
    return _ParallelFn.apply(x, layer, peers, sp, grad_peers, copy_out)


def sp_rows(x: torch.Tensor, world: int) -> int:
    """Tokens per rank of a sequence-parallel activation ``x[s, ..., features]``: the flattened rows
    ``[r*M/world, (r+1)*M/world)`` belong to rank r, which needs ``x.shape[0] % world == 0``."""
    if x.dim() < 2 or x.shape[0] % world != 0:
        raise ValueError(f"sequence parallelism splits the first dimension of the activation over the ranks: "
                         f"{tuple(x.shape)} does not split over a world of {world}")
    return x.numel() // x.shape[-1] // world


def _group_world_rank(group) -> tuple[int, int]:
    if dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


def _gather_columns(layer, inp, M: int, dtype: torch.dtype, device, **kw) -> torch.Tensor:
    """The ``[M, world * rows]`` output of a column-parallel layer: ``layer.local_forward`` (given ``kw``) writes this
    rank's ``[M, rows]`` block into its slot of a ``[world, M, rows]`` stage (kept on the layer for the next call), and
    the stage is all-gathered.  The blocks sit side by side along the inner dimension of a row-major matrix, which
    ``all_gather_into_tensor`` cannot write in place, hence the stage and the permute."""
    world, rank = _group_world_rank(layer.group)
    rows = layer.shard.rows
    stage = layer._stage
    if stage is None or stage.shape != (world, M, rows) or stage.dtype != dtype or stage.device != device:
        stage = layer._stage = torch.empty((world, M, rows), device=device, dtype=dtype)
    layer.local_forward(inp, stage[rank], rows, **kw)
    dist.all_gather_into_tensor(stage.view(-1), stage[rank].reshape(-1), group=layer.group)
    return stage.permute(1, 0, 2).reshape(M, world * rows)


def _check_peers(peers, M: int, N: int, dtype: torch.dtype, what: str) -> None:
    """``peers`` (a :class:`PeerGather` or :class:`PeerPartials`) was built for ``[M, N]`` of ``dtype``: checked on the
    host before any launch."""
    if M != peers.M or N != peers.N or dtype != peers.dtype:
        raise ValueError(f"{type(peers).__name__} was built for a different {what}")


def _gather_partials(layer, inp, M: int, dtype: torch.dtype, device, what: str, **kw) -> torch.Tensor:
    """The ``[world, M, N]`` partials of a row-parallel layer: ``layer.partial_forward`` (given ``kw``) writes this
    rank's into its slot of a stage (kept on the layer for the next call), and the stage is all-gathered."""
    world, rank = _group_world_rank(layer.group)
    stage = layer._stage
    if stage is None or stage.shape[:2] != (world, M) or stage.device != device:
        stage = layer._stage = torch.empty((world, M, layer.shard.rows), device=device, dtype=dtype)
    if not layer.partial_forward(inp, [stage[rank]], **kw):
        raise RuntimeError(f"{what} does not serve this shard shape")
    if world > 1:
        dist.all_gather_into_tensor(stage.view(-1), stage[rank].reshape(-1), group=layer.group)
    return stage


def _sp_exchange(layer, inp, Ms: int, dtype: torch.dtype, what: str) -> torch.Tensor:
    """A sequence-parallel row layer's ``[world, M/world, N]`` partials of this rank's tokens, chunk r from rank r:
    ``layer.partial_forward`` writes the full ``[M, N]`` partial of ``dtype`` into a send buffer (kept on the layer with
    its receive buffer for the next call), then an all-to-all (NCCL's reduce-scatter would sum in another order)."""
    world, _ = _group_world_rank(layer.group)
    shape = (world, Ms, layer.shard.rows)
    bufs = layer._sp_bufs
    if bufs is None or bufs[0].shape != shape or bufs[0].device != inp.device:
        bufs = layer._sp_bufs = tuple(torch.empty(shape, device=inp.device, dtype=dtype) for _ in range(2))
    send, recv = bufs
    if not layer.partial_forward(inp, [send]):
        raise RuntimeError(f"{what} does not serve this shard shape")
    if world == 1:
        return send
    dist.all_to_all_single(recv, send, group=layer.group)
    return recv


class _PeerSlots:
    """Two symmetric-memory buffers of ``shape`` shared by the ranks of ``group``, used in turn, so that a rank may
    start step i + 1 while a peer still reads step i."""

    def __init__(self, shape, dtype: torch.dtype, device, group: Optional[dist.ProcessGroup]):
        import torch.distributed._symmetric_memory as symm_mem

        group = group if group is not None else dist.group.WORLD
        self.dtype = dtype
        self.bufs, self.handles = [], []
        for _ in range(2):
            t = symm_mem.empty(shape, dtype=dtype, device=device)
            self.handles.append(symm_mem.rendezvous(t, group))
            self.bufs.append(t)
        self.world = self.handles[0].world_size
        self.rank = self.handles[0].rank
        self.step = 0

    def slot(self):
        """(local tensor, [base address of that slot on rank r for every r], handle) of the next step."""
        i = self.step & 1
        self.step += 1
        return self.bufs[i], [int(p) for p in self.handles[i].buffer_ptrs], self.handles[i]

    def dest_ptrs(self, bases, offset: int) -> list[int]:
        """The address ``offset`` bytes into every rank's buffer of a slot (``bases`` from :meth:`slot`): this rank's
        own buffer first, as the multi-destination GEMMs take their local output, then the peers in rank order."""
        return [bases[r] + offset for r in [self.rank] + [r for r in range(self.world) if r != self.rank]]

    def scatter_ptrs(self, bases, offset: int) -> list[int]:
        """The address ``offset`` bytes into every rank's buffer of a slot, in rank order, as the scatter GEMM takes its
        destinations (rank s's rows to rank s)."""
        return [bases[r] + offset for r in range(self.world)]


class PeerGather(_PeerSlots):
    """Two symmetric-memory ``[M, N]`` output slots shared by the ranks of ``group``."""

    def __init__(self, M: int, N: int, dtype: torch.dtype, device, group: Optional[dist.ProcessGroup] = None):
        super().__init__((M, N), dtype, device, group)
        self.M, self.N = M, N


class PeerInputGrad(_PeerSlots):
    """Two symmetric-memory ``[M, F]`` slots of ``dtype`` through which the backward of a fused route exchanges (pass it
    as ``grad_peers``); allocate it once, outside a timed or captured step, as :class:`PeerGather`.

    * column layer (``fused_forward``, ``fused_forward_col8`` and their ``_sp`` forms): fp32 ``[M, K]``, M all tokens.
      Rank r stores its partial ``P_r = G_r . W_r`` into its own slot, one barrier, and each rank reduces the peers'
      slots in rank order (``reduce_partials_ptrs``): all M rows, or only its own tokens' rows under sequence
      parallelism -- a reduce-scatter by pull, with the bits of the ``all_to_all_single`` route.
    * row layer, sequence parallel: ``[M, N]`` of the activation dtype; rank r copies its tokens' rows of ``grad_y``
      into its rows of every rank's slot, one barrier, then ``G . W_r``.
    * row layer, ``input_is_parallel=False``: ``[M, in_features]`` of the activation dtype; rank r copies its
      ``grad_x_r`` into its columns ``[k0, k0 + K/w)`` of every rank's slot, one barrier.  The gradient is a copy of the
      slot, which the peers rewrite two exchanges later.
    * row layer, ``input_is_parallel=True`` without sequence parallelism: no exchange; only the group is checked.

    Reuse: a rank writes slot i (its own, or its rows / columns of the peers') again only two exchanges later, after the
    barrier of the exchange in between, which no peer reaches before its reads of slot i -- enqueued earlier on its
    stream -- have completed."""

    def __init__(self, M: int, F: int, dtype: torch.dtype, device, group: Optional[dist.ProcessGroup] = None):
        super().__init__((M, F), dtype, device, group)
        self.M, self.F = M, F
        self.group = group


def _check_peer_grad(peers, group, shape=None, dtype: Optional[torch.dtype] = None) -> None:
    """``peers`` is a :class:`PeerInputGrad` of ``group`` and, when ``shape`` is given, of that slot shape and dtype."""
    if not isinstance(peers, PeerInputGrad):
        raise ValueError(f"grad_peers must be a PeerInputGrad, got {type(peers).__name__}")
    world = dist.group.WORLD if dist.is_initialized() else None
    if (peers.group if peers.group is not None else world) is not (group if group is not None else world):
        raise ValueError("grad_peers was built for another process group than the layer's")
    if shape is not None and ((peers.M, peers.F) != tuple(shape) or peers.dtype != dtype):
        raise ValueError(f"PeerInputGrad was built for [{peers.M}, {peers.F}] {peers.dtype}; this backward exchanges "
                         f"{list(shape)} {dtype}")


def fused_forward(layer: "ColumnParallelLinear4bit", x: torch.Tensor, peers: PeerGather,
                  grad_peers: Optional[PeerInputGrad] = None) -> torch.Tensor:
    """``layer(x)`` with the all-gather fused into the GEMM epilogue; returns this rank's [M, N] slot, valid until the
    slot comes round again two calls later.  With ``grad_peers = PeerInputGrad(M, K, torch.float32)`` an input that
    requires grad gets its gradient, exchanged through symmetric memory, and the call returns a copy of the slot, which
    autograd may keep until the backward."""
    return _fused_route("fused_forward", layer, x, peers, False, grad_peers, copy_out=True)


def _ftz(t: torch.Tensor) -> torch.Tensor:
    """fp32 values below the normal range flushed to (signed) zero, as the kernels' ``mul.ftz`` does."""
    return torch.where(t.abs() < 2.0**-126, t * 0.0, t)


def nested_scales(qs: F.QuantState) -> torch.Tensor:
    """The fp32 scale of every quantisation block of a double-quantised state, computed as the kernels fetch it
    (``ScaleSrc::load_as``): ``(code2[absmax_8bit] * absmax2[block // 256])`` rounded, flushed to zero below the
    normal range, then ``+ offset`` rounded."""
    return _nested_scales(qs.absmax, qs.state2.absmax, qs.state2.code, qs.offset)


def _nested_scales(absmax_8bit, absmax2, code, offset) -> torch.Tensor:
    a2 = absmax2.float()
    idx = torch.arange(absmax_8bit.numel(), device=a2.device) // 256
    prod = _ftz(_ftz(code.float()[absmax_8bit.long()]) * _ftz(a2[idx]))
    return prod + offset.reshape(()).float().to(prod.device)


def slice_quantized_weight_k(packed: torch.Tensor, qs: F.QuantState, world: int, rank: int) -> Shard4bit:
    """Cut rank's input features ``W[:, k0:k1]`` out of a weight quantised once, globally (no re-quantisation).

    The slice is strided in the packed layout (``[N, K/2]`` bytes, ``[N, K/blocksize]`` absmax), so the shard is a
    repacked copy, made once at load.  Requires ``K % (world * blocksize) == 0`` and ``(K / world) % 64 == 0`` (the
    shard stays on the tensor-core kernels).  A double-quantised state's level-2 groups of 256 blocks straddle the
    shards, so the shard's scales are plain fp32 absmax computed exactly as the kernels fetch the nested ones
    (:func:`nested_scales`): the shard decodes to the same weights bit for bit."""
    N, K = qs.shape
    bs = qs.blocksize
    _check_rank(world, rank)
    if K % (world * bs) != 0:
        raise ValueError(f"in_features ({K}) must be a multiple of world * blocksize ({world} * {bs}) to shard by "
                         "input features")
    kr = K // world
    if kr % 64 != 0:
        raise ValueError(f"in_features per shard ({kr}) must be a multiple of 64")
    k0 = rank * kr
    flat = packed.reshape(-1).view(torch.uint8) if packed.dtype != torch.uint8 else packed.reshape(-1)
    codes = flat[:N * K // 2].view(N, K // 2)[:, k0 // 2:(k0 + kr) // 2].contiguous().view(-1)
    scales = nested_scales(qs) if qs.nested else qs.absmax
    absmax = scales.reshape(N, K // bs)[:, k0 // bs:(k0 + kr) // bs].contiguous().view(-1)
    return Shard4bit(packed=codes, absmax=absmax, absmax_8bit=None, absmax_code=None, absmax_offset=None, rows=N,
                     row0=0, K=kr, blocksize=bs, quant_type=qs.quant_type, k0=k0)


class RowParallelLinear4bit(_RowInputGrad, torch.nn.Module):
    """``y = x @ dequant(W)^T + b`` with W's input features split across the process group: every rank returns the
    whole ``[..., N]`` output, the same bits on every rank."""

    def __init__(self, shard: Shard4bit, in_features: int, bias: Optional[torch.Tensor] = None,
                 group: Optional[dist.ProcessGroup] = None, input_is_parallel: bool = True,
                 sequence_parallel: bool = False):
        super().__init__()
        self.shard = shard
        self.in_features = in_features
        self.out_features = shard.rows
        self.group = group
        self.input_is_parallel = input_is_parallel
        self.sequence_parallel = sequence_parallel
        self.bias = None if bias is None else bias.contiguous()
        self._stage = None
        self._sp_bufs = None

    @classmethod
    def from_quantized(cls, packed, qs: F.QuantState, bias=None, group=None, input_is_parallel=True,
                       sequence_parallel=False):
        world, rank = _group_world_rank(group)
        return cls(slice_quantized_weight_k(packed, qs, world, rank), qs.shape[1], bias, group, input_is_parallel,
                   sequence_parallel)

    def local_input(self, x: torch.Tensor) -> torch.Tensor:
        """This rank's ``x_r[..., K/world]``: ``x`` itself, or its slice when the layer takes the full input."""
        s = self.shard
        if self.input_is_parallel:
            if x.shape[-1] != s.K:
                raise ValueError(f"expected this rank's {s.K} input features, got {x.shape[-1]}")
            return x
        if x.shape[-1] != self.in_features:
            raise ValueError(f"expected {self.in_features} input features, got {x.shape[-1]}")
        return x[..., s.k0:s.k0 + s.K]

    def partial_forward(self, x_r: torch.Tensor, outs, ldc: Optional[int] = None) -> bool:
        """``P_r = x_r . dequant(W_r)^T`` in fp32 (no bias, no rounding) to every destination in ``outs``."""
        s = self.shard
        return gemm_4bit_partial(x_r, s.packed, (s.rows, s.K), s.absmax, s.blocksize, s.quant_type, None, None, None,
                                 outs, s.rows if ldc is None else ldc)

    def partial_scatter(self, x_r: torch.Tensor, outs, ldc: Optional[int] = None) -> bool:
        """:meth:`partial_forward` with the rows of ``P_r`` split over ``outs`` in rank order: rank s's tokens go to
        ``outs[s]`` (sequence parallelism)."""
        s = self.shard
        return gemm_4bit_partial_scatter(x_r, s.packed, (s.rows, s.K), s.absmax, s.blocksize, s.quant_type, None, None,
                                         None, outs, s.rows if ldc is None else ldc)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _ParallelFn.apply(x, self)

    def _forward(self, x: torch.Tensor, peers: Optional["PeerPartials"] = None,
                 sp: Optional[bool] = None) -> torch.Tensor:
        """The layer's output.  ``sp`` (default: ``sequence_parallel``) chooses the mode.  With ``peers`` the partials
        are exchanged through its symmetric-memory slot, followed by one barrier: the GEMM epilogue stores ``P_r`` into
        slot r of every rank's buffer or, under sequence parallelism, the rows of rank s's tokens into slot r of rank
        s's buffer (the NCCL exchange filling the slot when the scatter GEMM refuses the call)."""
        s = self.shard
        world, _ = _group_world_rank(self.group)
        x_r = self.local_input(x)
        if self.sequence_parallel if sp is None else sp:
            Ms = sp_rows(x_r, world)
            lead = (x_r.shape[0] // world, *x_r.shape[1:-1])
            if peers is None:
                parts = _sp_exchange(self, x_r, Ms, torch.float32, "gemm_4bit_partial")
            else:
                _check_peers(peers, Ms, s.rows, torch.float32, "output shape or dtype")
                parts, bases, handle = peers.slot()
                if not self.partial_scatter(x_r, peers.scatter_ptrs(bases, peers.rank * Ms * s.rows * 4)):
                    # the scatter GEMM refused the call: the NCCL route fills the slot
                    parts.copy_(_sp_exchange(self, x_r, Ms, torch.float32, "gemm_4bit_partial"))
                handle.barrier(channel=0)  # every rank's rows have landed at their owner
        else:
            M = x_r.numel() // s.K
            lead = x_r.shape[:-1]
            if peers is None:
                parts = _gather_partials(self, x_r, M, torch.float32, x_r.device, "gemm_4bit_partial")
            else:
                _check_peers(peers, M, s.rows, torch.float32, "output shape or dtype")
                parts, bases, handle = peers.slot()
                if not self.partial_forward(x_r, peers.dest_ptrs(bases, peers.rank * M * s.rows * 4)):
                    raise RuntimeError("gemm_4bit_partial does not serve this shard shape")
                handle.barrier(channel=0)  # every rank's partial has landed everywhere
        return reduce_partials(parts, x_r.dtype, self.bias).view(*lead, s.rows)


class PeerPartials(_PeerSlots):
    """Two symmetric-memory ``[world, M, N]`` partial slots shared by the ranks of ``group`` (fp32 for the 4-bit layer,
    int32 for the int8 one)."""

    def __init__(self, M: int, N: int, device, group: Optional[dist.ProcessGroup] = None,
                 dtype: torch.dtype = torch.float32):
        world, _ = _group_world_rank(group)
        super().__init__((world, M, N), dtype, device, group)
        self.M, self.N = M, N


def fused_forward_row(layer: RowParallelLinear4bit, x: torch.Tensor, peers: PeerPartials,
                      grad_peers: Optional[PeerInputGrad] = None) -> torch.Tensor:
    """``layer(x)`` with the exchange of the partials fused into the GEMM epilogue: ``P_r`` is stored into slot r of
    every rank's buffer, one barrier publishes them, and each rank reduces them in rank order.  With ``grad_peers``
    an input that requires grad gets its gradient, exchanged through symmetric memory."""
    return _fused_route("fused_forward_row", layer, x, peers, False, grad_peers)


def fused_forward_row_sp(layer: RowParallelLinear4bit, x: torch.Tensor, peers: PeerPartials,
                         grad_peers: Optional[PeerInputGrad] = None) -> torch.Tensor:
    """The sequence-parallel ``layer(x)`` (this rank's tokens only) with the reduce-scatter fused into the GEMM
    epilogue: the rows of ``P_r`` that belong to rank s are stored into slot r of rank s's ``[world, M/world, N]``
    buffer (``peers = PeerPartials(M // world, N)``), one barrier publishes them, and each rank reduces its own.  With
    ``grad_peers = PeerInputGrad(M, N, x.dtype)`` an input that requires grad gets its gradient: the token rows of
    ``grad_y`` gathered through symmetric memory."""
    return _fused_route("fused_forward_row_sp", layer, x, peers, True, grad_peers)


def fused_forward_col_sp(layer: ColumnParallelLinear4bit, x: torch.Tensor, peers: PeerGather,
                         grad_peers: Optional[PeerInputGrad] = None) -> torch.Tensor:
    """The sequence-parallel ``layer(x)`` with the token all-gather through symmetric memory: this rank copies its
    ``[M/world, ..., K]`` tokens into its rows of every rank's ``[M, K]`` buffer (``peers = PeerGather(M, K, dtype)``),
    one barrier publishes them, and the local GEMM reads the gathered tokens.  Returns ``[M, ..., N/world]``.  With
    ``grad_peers = PeerInputGrad(M, K, torch.float32)`` an input that requires grad gets the gradient of its tokens,
    reduced from the peers' partials."""
    return _fused_route("fused_forward_col_sp", layer, x, peers, True, grad_peers)


def reassemble_shards(shards: list[Shard4bit]) -> tuple[torch.Tensor, torch.Tensor]:
    """Inverse of slice_quantized_weight for the plain (non-nested) case: (packed, absmax)."""
    return torch.cat([s.packed for s in shards]), torch.cat([s.absmax for s in shards])


# ====================================================================================== tensor-parallel expert layers
# Mixture-of-experts layers on a 4-bit [E, N, K] expert tensor (GroupedLinear4bit's weight, quantised once, globally),
# sharded as the dense layers are: the column layer (gate_up) holds output rows [r*N/w, (r+1)*N/w) of EVERY expert, the
# row layer (down) input features [r*K/w, (r+1)*K/w) of every expert.  Routing stays with the model: each layer takes
# the expert-sorted rows x [M, K] and the int32 end row of every expert, offs [E], on the device.  ``offs`` and the token
# rows must be the same on every rank.  Nothing reads offs on the host, so a forward can be captured in a CUDA graph.
#   * column: one grouped GEMM on the shard (the unsharded kernel and tile on fewer rows per expert), so the gathered
#     output is GroupedLinear4bit's bit for bit.
#   * row: the grouped fp32 partial of the shard (the unsharded layer's tile, which depends on M and E only), the
#     partials gathered as the dense row layer gathers them, and a rank-order reduction that adds each row's expert
#     bias and rounds once.  With one rank that is GroupedLinear4bit's output bit for bit; with more it differs only by
#     the order of the fp32 sum.
# Inference only: an input that requires grad, sequence parallelism and the symmetric-memory routes are refused.

def slice_grouped_weight(packed: torch.Tensor, qs: F.QuantState, world: int, rank: int) -> Shard4bit:
    """Cut rank's output rows ``[r*N/w, (r+1)*N/w)`` out of every expert of an ``[E, N, K]`` expert tensor quantised
    once, globally, and stack them as an ``[E, N/w, K]`` shard.  Requires ``K % blocksize == 0`` and ``N % world == 0``.
    Nested statistics stay nested when every expert's slice starts and ends on a 256-block boundary; otherwise they
    become plain fp32 scales computed as the kernels fetch them (:func:`nested_scales`), which decode to the same
    weights bit for bit.

    A fused ``gate_up`` tensor that stacks gate and up along N is cut into contiguous N ranges, so the slice of a rank
    holds matching gate and up rows only if the tensor interleaves them that way; the layer does not reorder."""
    if len(qs.shape) != 3:
        raise ValueError(f"slice_grouped_weight: the state must be of an [E, N, K] expert tensor, got {list(qs.shape)}")
    E, N, K = qs.shape
    bs = qs.blocksize
    _check_rank(world, rank)
    if K % bs != 0:
        raise ValueError(f"in_features ({K}) must be a multiple of the blocksize ({bs}) to shard by rows")
    row0, rows = shard_rows(N, world, rank)
    flat = packed.reshape(-1).view(torch.uint8) if packed.dtype != torch.uint8 else packed.reshape(-1)
    codes = flat[:E * N * K // 2].view(E, N * K // 2)[:, row0 * K // 2:(row0 + rows) * K // 2].contiguous().view(-1)
    nb = N * K // bs  # quantisation blocks per expert
    a0, a1 = row0 * K // bs, (row0 + rows) * K // bs
    common = dict(rows=rows, row0=row0, K=K, blocksize=bs, quant_type=qs.quant_type, experts=E)
    if qs.nested and all((e * nb + a0) % 256 == 0 for e in range(E)) and (a1 - a0) % 256 == 0:
        a2 = torch.cat([qs.state2.absmax[(e * nb + a0) // 256:(e * nb + a1) // 256] for e in range(E)])
        return Shard4bit(packed=codes, absmax=a2, absmax_8bit=qs.absmax.reshape(E, nb)[:, a0:a1].contiguous().view(-1),
                         absmax_code=qs.state2.code, absmax_offset=qs.offset.reshape(1).float(), **common)
    scales = nested_scales(qs) if qs.nested else qs.absmax
    return Shard4bit(packed=codes, absmax=scales.reshape(E, nb)[:, a0:a1].contiguous().view(-1), absmax_8bit=None,
                     absmax_code=None, absmax_offset=None, **common)


def slice_grouped_weight_k(packed: torch.Tensor, qs: F.QuantState, world: int, rank: int) -> Shard4bit:
    """Rank's input features ``[r*K/w, (r+1)*K/w)`` of every expert of an ``[E, N, K]`` expert tensor:
    :func:`slice_quantized_weight_k` of the flattened ``[E*N, K]`` weight (the same rules; plain fp32 scales), as an
    ``[E, N, K/w]`` shard."""
    if len(qs.shape) != 3:
        raise ValueError(f"slice_grouped_weight_k: the state must be of an [E, N, K] expert tensor, got "
                         f"{list(qs.shape)}")
    E, N, K = qs.shape
    flat = F.QuantState(absmax=qs.absmax, shape=torch.Size([E * N, K]), code=qs.code, blocksize=qs.blocksize,
                        quant_type=qs.quant_type, dtype=qs.dtype, offset=qs.offset, state2=qs.state2)
    s = slice_quantized_weight_k(packed, flat, world, rank)
    s.rows, s.experts = N, E
    return s


def _grouped_inference_only(what: str, x: torch.Tensor) -> None:
    if torch.is_grad_enabled() and x.requires_grad:
        raise RuntimeError(f"{what} is inference only: the input requires grad, and training through the tensor-parallel "
                           "expert layers is not implemented (run it under torch.no_grad() or detach the input)")


class _GroupedNoFusedRoute:
    """The fused symmetric-memory routes (``fused_forward*``) call ``_forward`` / ``_grad_slot``: refused."""

    def _refuse(self, *args, **kwargs):
        raise RuntimeError(f"{type(self).__name__} has no symmetric-memory route: call the layer itself")

    _forward = _grad_slot = _refuse


def _no_sequence_parallel(cls, sequence_parallel: bool) -> None:
    if sequence_parallel:
        raise ValueError(f"{cls.__name__} does not support sequence_parallel=True")


class ColumnParallelGroupedLinear4bit(_GroupedNoFusedRoute, torch.nn.Module):
    """The experts of a mixture-of-experts layer with their output features split across the process group (gate_up):
    ``forward(x, offs)`` gives this rank's ``[M, N/w]`` columns, or with ``gather_output`` the whole ``[M, N]``,
    GroupedLinear4bit's output bit for bit.  ``bias`` is the full ``[E, N]`` bias, of which the layer keeps its
    ``[E, N/w]`` slice.  See :func:`slice_grouped_weight` for fused gate_up tensors."""

    def __init__(self, shard: Shard4bit, out_features: int, bias: Optional[torch.Tensor] = None,
                 group: Optional[dist.ProcessGroup] = None, gather_output: bool = True, sequence_parallel: bool = False):
        super().__init__()
        _no_sequence_parallel(type(self), sequence_parallel)
        self.shard = shard
        self.out_features = out_features
        self.group = group
        self.gather_output = gather_output
        self.bias_shard = None if bias is None else \
            bias.reshape(shard.experts, out_features)[:, shard.row0:shard.row0 + shard.rows].contiguous()
        self._stage = None

    @classmethod
    def from_quantized(cls, packed, qs: F.QuantState, bias=None, group=None, gather_output=True,
                       sequence_parallel=False):
        world, rank = _group_world_rank(group)
        return cls(slice_grouped_weight(packed, qs, world, rank), qs.shape[1], bias, group, gather_output,
                   sequence_parallel)

    def local_forward(self, x: torch.Tensor, out: Optional[torch.Tensor] = None, ldc: Optional[int] = None, *,
                      offs: torch.Tensor) -> torch.Tensor:
        """This rank's ``[M, N/w]`` columns; written into ``out`` (row stride ``ldc`` elements) if given."""
        s = self.shard
        if out is None:
            out = torch.empty((x.shape[0], s.rows), device=x.device, dtype=x.dtype)
            ldc = s.rows
        gemm_4bit_grouped_into(x, s.packed, (s.experts, s.rows, s.K), s.absmax, s.blocksize, s.quant_type, offs,
                               self.bias_shard, s.absmax_8bit, s.absmax_code, s.absmax_offset, out, ldc)
        return out

    def forward(self, x: torch.Tensor, offs: torch.Tensor) -> torch.Tensor:
        _grouped_inference_only(type(self).__name__, x)
        world, _ = _group_world_rank(self.group)
        if world == 1 or not self.gather_output:
            return self.local_forward(x, offs=offs)
        return _gather_columns(self, x, x.shape[0], x.dtype, x.device, offs=offs)


class RowParallelGroupedLinear4bit(_GroupedNoFusedRoute, torch.nn.Module):
    """The experts of a mixture-of-experts layer with their input features split across the process group (down):
    ``forward(x, offs)`` returns the whole ``[M, N]`` output, the same bits on every rank.  Each rank computes the fp32
    partial of its K slice for every expert (no bias, no rounding), the partials are all-gathered, and every rank sums
    them in rank order, adds the bias of each row's expert (``bias`` ``[E, N]``) and rounds once."""

    def __init__(self, shard: Shard4bit, in_features: int, bias: Optional[torch.Tensor] = None,
                 group: Optional[dist.ProcessGroup] = None, input_is_parallel: bool = True,
                 sequence_parallel: bool = False):
        super().__init__()
        _no_sequence_parallel(type(self), sequence_parallel)
        self.shard = shard
        self.in_features = in_features
        self.out_features = shard.rows
        self.group = group
        self.input_is_parallel = input_is_parallel
        self.bias = None if bias is None else bias.reshape(shard.experts, shard.rows).contiguous()
        self._stage = None

    @classmethod
    def from_quantized(cls, packed, qs: F.QuantState, bias=None, group=None, input_is_parallel=True,
                       sequence_parallel=False):
        world, rank = _group_world_rank(group)
        return cls(slice_grouped_weight_k(packed, qs, world, rank), qs.shape[2], bias, group, input_is_parallel,
                   sequence_parallel)

    local_input = RowParallelLinear4bit.local_input

    def partial_forward(self, x_r: torch.Tensor, outs, ldc: Optional[int] = None, *, offs: torch.Tensor) -> bool:
        """``P_r = x_r . dequant(W_r)^T`` of every expert's rows in fp32 (no bias, no rounding) into ``outs[0]``."""
        s = self.shard
        if len(outs) != 1:
            raise ValueError("the grouped partial GEMM writes one destination")
        gemm_4bit_grouped_partial(x_r, s.packed, (s.experts, s.rows, s.K), s.absmax, s.blocksize, s.quant_type, offs,
                                  outs[0], s.rows if ldc is None else ldc)
        return True

    def forward(self, x: torch.Tensor, offs: torch.Tensor) -> torch.Tensor:
        _grouped_inference_only(type(self).__name__, x)
        x_r = self.local_input(x)
        parts = _gather_partials(self, x_r, x_r.shape[0], torch.float32, x_r.device, "gemm_4bit_grouped_partial",
                                 offs=offs)
        return reduce_partials_grouped(parts, offs, x_r.dtype, self.bias)


# ====================================================================================== tensor-parallel LLM.int8()
# Column and row sharding of the inference Linear8bitLt (``has_fp16_weights=False``).  The weight is quantised once,
# globally (CB [N, K] int8, SCB [N] fp32 row absmax) and every shard is a slice of it.  Both layers return, on every
# rank, the unsharded layer's output bit for bit:
#   * column (rank r owns output rows [r*N/w, (r+1)*N/w)): every rank quantises the replicated x exactly as the
#     unsharded layer does and runs the same GEMM on its rows; each output element's epilogue depends only on its own
#     row and column, so the slices are the unsharded output's columns.
#   * row (rank r owns input features [k0, k1)): the statistics of x are combined before quantising (the row absmax is
#     a max over the ranks' slices), the int32 partials CA_r . CB_r^T add up exactly to the unsharded accumulator, and
#     the reduction applies the GEMM's own per-element epilogue once.  The outlier columns of the ranks, concatenated
#     in rank order, are the unsharded ascending list, and their operands are the unsharded ones.
# Beyond 64 outlier columns the unsharded layer adds the outlier product with `addmm`; both layers then run that same
# `addmm` on the same full-size operands.  ``state.idx`` is not kept.
#
# Training (LoRA on an 8-bit base).  Both layers run their forward through ``_ParallelFn`` (the same bits) and share the
# 4-bit layers' backward (``_ColumnInputGrad`` / ``_RowInputGrad``): the input gradient ``grad_y . W`` and nothing else,
# W = T(CB * SCB / 127) dequantised in one pass (``Shard8bit.dequantize``) as ``MatMul8bitLt.backward`` dequantises it.
# As there, the outlier decomposition of the forward leaves the gradient alone: the whole CB enters it, so the backward
# needs no outlier list and no host synchronisation.
#
# Sequence parallelism (``sequence_parallel=True``, as for the 4-bit layers: rank r owns the flattened tokens
# ``[r*M/w, (r+1)*M/w)`` of an activation whose first dimension splits over the ranks).  The outputs stay the unsharded
# bits: the column layer returns ``[M, ..., N/w]``, the row layer its tokens' rows ``[M/w, ..., N]``.
#   * column: LLM.int8() quantises each token on its own except for the zeroing of the outlier columns, so a rank
#     quantises only its tokens, the ranks agree on the outlier columns (an all-reduce MAX of the flags) and zero them,
#     and the int8 codes, the row statistics and the outlier columns of x are all-gathered instead of the activations:
#     half the bytes of fp16 / bf16, and 1/w of the quantisation work.  Needs ``gather_output=False`` and K % 16 == 0.
#   * row: the prologue is unchanged; the outlier counts are gathered before the GEMM, so every rank knows which route
#     runs before any partial is stored.  Up to 64 outlier columns, the int32 partial's rows go to the ranks that own
#     them (``all_to_all_single``, or the scatter GEMM into symmetric memory) and each rank reduces its ``[w, M/w, N]``
#     with its rows of SCA and subA: the reduction works element by element, so these are the unsharded rows.  Past 64,
#     an `addmm` on M/w rows need not give the bits of the one on M rows, so both routes run the non-SP computation and
#     keep their rows: the slow path, with the non-SP exchange and reduction.

_INT8_FUSED_J = 64  # outlier columns the GEMM epilogue takes; beyond, the unsharded layer runs the addmm chain


@dataclass
class Shard8bit:
    """The slice of a globally quantised int8 weight owned by one rank."""

    CB: torch.Tensor   # int8 [rows, K] (row shard) | [N, K / world] (K shard)
    SCB: torch.Tensor  # fp32 [rows] (row shard) | [N], replicated (K shard)
    rows: int
    row0: int
    K: int
    k0: int = 0

    def dequantize(self, dtype: torch.dtype) -> torch.Tensor:
        """The shard's weight ``[rows, K]`` in ``dtype`` (fp16 / bf16) as ``MatMul8bitLt.backward`` dequantises it,
        ``dtype(CB * (SCB / 127))`` row by row, in one pass (``int8_dequant_rows``)."""
        return int8_dequant_rows(self.CB, self.SCB, dtype)


def _check_rank(world: int, rank: int) -> None:
    if world < 1 or not 0 <= rank < world:
        raise ValueError(f"rank {rank} outside a world of {world}")


def slice_int8_weight(CB: torch.Tensor, SCB: torch.Tensor, world: int, rank: int) -> Shard8bit:
    """Rank's output rows ``CB[n0:n1]`` and ``SCB[n0:n1]`` of a weight quantised once, globally."""
    _check_rank(world, rank)
    N, K = CB.shape
    row0, rows = shard_rows(N, world, rank)
    return Shard8bit(CB=CB[row0:row0 + rows].contiguous(), SCB=SCB[row0:row0 + rows].contiguous(), rows=rows,
                     row0=row0, K=K)


def slice_int8_weight_k(CB: torch.Tensor, SCB: torch.Tensor, world: int, rank: int) -> Shard8bit:
    """Rank's input features ``CB[:, k0:k1]`` (repacked once) of a weight quantised once, globally.  ``SCB`` is the
    full-row absmax and stays replicated.  Requires ``K % (16 * world) == 0``, so that every shard stays on the int8
    GEMM."""
    _check_rank(world, rank)
    N, K = CB.shape
    if K % (16 * world) != 0:
        raise ValueError(f"in_features ({K}) must be a multiple of 16 * world ({16 * world}) to shard by input features")
    kr = K // world
    k0 = rank * kr
    return Shard8bit(CB=CB[:, k0:k0 + kr].contiguous(), SCB=SCB.contiguous(), rows=N, row0=0, K=kr, k0=k0)


def _state_of(module) -> tuple[torch.Tensor, torch.Tensor, float]:
    """(CB, SCB, threshold) of an inference Linear8bitLt on the GPU."""
    if module.state.has_fp16_weights:
        raise ValueError("the tensor-parallel int8 layers shard an inference Linear8bitLt (has_fp16_weights=False)")
    CB = module.state.CB if module.state.CB is not None else module.weight.CB
    SCB = module.state.SCB if module.state.SCB is not None else module.weight.SCB
    if CB is None or SCB is None:
        raise ValueError("the Linear8bitLt is not quantised yet: move it to the GPU first")
    return CB, SCB, float(module.state.threshold)


def _no_capture(threshold: float, what: str) -> None:
    if threshold > 0.0 and torch.cuda.is_current_stream_capturing():
        raise RuntimeError(f"{what}: threshold > 0 needs the outlier count on the host and cannot run under CUDA-graph "
                           "capture; capture with threshold 0")


@dataclass
class Int8Input:
    """The activations of a column-parallel layer quantised as the unsharded layer quantises them."""

    A: Optional[torch.Tensor]  # [M, K] of the input dtype; None with sequence parallelism (only subA is gathered)
    CA: torch.Tensor      # int8 [M, K], outlier columns zeroed
    SCA: torch.Tensor     # fp32 [M]
    cols: Optional[torch.Tensor]  # int64 ascending outlier columns, or None
    dtype: torch.dtype    # the input dtype
    # sequence parallelism, gathered over the ranks: x[:, cols] zero-padded to [M, jpad] with this rank's subBT
    # [rows, jpad] (J <= 64: the GEMM's outlier operands), or [M, J] (J > 64: the addmm operand)
    subA: Optional[torch.Tensor] = None
    subBT: Optional[torch.Tensor] = None

    @property
    def J(self) -> int:
        return 0 if self.cols is None else int(self.cols.numel())


class ColumnParallelLinear8bitLt(_ColumnInputGrad, torch.nn.Module):
    """LLM.int8() ``y = x @ W^T + b`` with W's output features split across the process group.  Every rank's output
    equals the unsharded inference ``Linear8bitLt`` output (its columns, with ``gather_output=False``) bit for bit.
    With ``sequence_parallel=True`` the input is this rank's tokens ``[M/w, ..., K]`` and the output ``[M, ..., N/w]``."""

    def __init__(self, shard: Shard8bit, out_features: int, bias: Optional[torch.Tensor] = None,
                 group: Optional[dist.ProcessGroup] = None, gather_output: bool = True, threshold: float = 0.0,
                 sequence_parallel: bool = False):
        super().__init__()
        if sequence_parallel and gather_output:
            raise ValueError("sequence_parallel=True hands each rank all tokens of its feature slice: it needs "
                             "gather_output=False")
        if sequence_parallel and shard.K % 16 != 0:
            raise ValueError(f"sequence_parallel=True gathers int8 codes for the int8 GEMM: in_features ({shard.K}) "
                             "must be a multiple of 16")
        self.shard = shard
        self.out_features = out_features
        self.group = group
        self.gather_output = gather_output
        self.threshold = float(threshold)
        self.sequence_parallel = sequence_parallel
        self.bias_shard = None if bias is None else bias[shard.row0:shard.row0 + shard.rows].contiguous()
        self._stage = None

    @classmethod
    def from_quantized(cls, CB, SCB, bias=None, group=None, threshold: float = 0.0, gather_output: bool = True,
                       sequence_parallel: bool = False):
        world, rank = _group_world_rank(group)
        return cls(slice_int8_weight(CB, SCB, world, rank), CB.shape[0], bias, group, gather_output, threshold,
                   sequence_parallel)

    @classmethod
    def from_linear8bitlt(cls, module, group=None, gather_output: bool = True, sequence_parallel: bool = False):
        CB, SCB, threshold = _state_of(module)
        return cls.from_quantized(CB, SCB, module.bias, group, threshold, gather_output, sequence_parallel)

    def _bias(self, dtype):
        b = self.bias_shard
        return None if b is None else b.to(dtype)

    def quantize(self, x: torch.Tensor) -> Int8Input:
        """x [..., K] -> the codes, statistics and outlier columns of the unsharded layer (the same on every rank)."""
        _no_capture(self.threshold, "ColumnParallelLinear8bitLt")
        A = x.reshape(-1, self.shard.K)
        CA, SCA, cols = F.int8_vectorwise_quant(A.to(torch.float16), threshold=self.threshold)
        return Int8Input(A, CA, SCA, cols if self.threshold > 0.0 else None, A.dtype)

    def local_quantize(self, x: torch.Tensor):
        """Sequence parallelism, step 1: (x_s [M/w, K], codes, row statistics, outlier flags or None) of this rank's
        tokens in one pass of the unsharded quantiser, the outlier columns not yet zeroed."""
        _no_capture(self.threshold, "ColumnParallelLinear8bitLt")
        xs = x.reshape(-1, self.shard.K)
        CA, SCA, flags = int8_vectorwise_quant_flags(xs.to(torch.float16), self.threshold)
        return xs, CA, SCA, flags

    def local_outliers(self, xs: torch.Tensor, CA: torch.Tensor, cols: Optional[torch.Tensor], M: int):
        """Sequence parallelism, step 3, given the outlier columns of all M tokens (the union of the ranks' flags): zeroes
        them in this rank's codes (for M > 1, as the unsharded quantiser does) and returns this rank's share of the
        outlier operands, (subA_s [M/w, jpad], subBT [rows, jpad]) up to 64 columns, (x_s[:, cols] [M/w, J], None)
        beyond, (None, None) without any."""
        J = 0 if cols is None else int(cols.numel())
        if J == 0:
            return None, None
        if M > 1:
            int8_zero_columns(CA, cols)
        if J <= _INT8_FUSED_J:
            return int8_outlier_operands(xs, self.shard.CB, self.shard.SCB, cols)
        return xs[:, cols].contiguous(), None

    def sp_quantize(self, x: torch.Tensor, peers: Optional["PeerInt8Input"] = None) -> Int8Input:
        """The quantised input of all M tokens from this rank's ``[M/w, ..., K]``: local quantisation, the outlier
        columns agreed by an all-reduce MAX of the flags (a host synchronisation, as in the unsharded layer), then the
        codes and row statistics all-gathered through NCCL or, with ``peers``, copied into this rank's rows of every
        rank's symmetric slot and published by one barrier.  The outlier columns of x travel through NCCL."""
        world, rank = _group_world_rank(self.group)
        K = self.shard.K
        Ms = x.numel() // K
        M = world * Ms
        if peers is not None and (peers.M != M or peers.K != K):
            raise ValueError("PeerInt8Input was built for a different token count / input width")
        xs, CA_s, SCA_s, flags = self.local_quantize(x)
        cols = None
        if flags is not None:
            if world > 1:
                dist.all_reduce(flags, op=dist.ReduceOp.MAX, group=self.group)
            cols = torch.nonzero(flags).view(-1)
        subA_s, subBT = self.local_outliers(xs, CA_s, cols, M)
        if peers is None:
            CA = torch.empty((M, K), device=x.device, dtype=torch.int8)
            SCA = torch.empty(M, device=x.device, dtype=torch.float32)
            dist.all_gather_into_tensor(CA, CA_s, group=self.group)
            dist.all_gather_into_tensor(SCA, SCA_s, group=self.group)
        else:
            local, _, handle = peers.slot()
            for r in range(world):
                handle.get_buffer(r, (Ms, K), torch.int8, rank * Ms * K).copy_(CA_s)
                handle.get_buffer(r, (Ms,), torch.float32, M * K // 4 + rank * Ms).copy_(SCA_s)
            handle.barrier(channel=0)  # every rank's codes and statistics have landed everywhere
            CA, SCA = peers.codes(local), peers.stats(local)
        subA = None
        if subA_s is not None:
            subA = torch.empty((M, subA_s.shape[1]), device=x.device, dtype=x.dtype)
            dist.all_gather_into_tensor(subA, subA_s, group=self.group)
        return Int8Input(None, CA, SCA, cols, x.dtype, subA, subBT)

    def local_forward(self, q: Int8Input, out: Optional[torch.Tensor] = None, ldc: Optional[int] = None):
        """This rank's [M, rows] columns of the unsharded output, without the outlier term past 64 columns (see
        :meth:`outlier_rows`); written into ``out`` (row stride ``ldc``) when given."""
        s = self.shard
        dtype = q.dtype
        M = q.CA.shape[0]
        if out is None:
            out = torch.empty((M, s.rows), device=q.CA.device, dtype=dtype)
            ldc = s.rows
        if not self._gemm(q, [out], ldc):
            if q.A is None:
                raise RuntimeError("the int8 GEMM does not serve this shard shape")
            # shapes the int8 GEMM does not take (K % 16): the library's own route, copied into place
            if 0 < q.J <= _INT8_FUSED_J:
                y, _ = torch.ops.bitsandbytes.int8_mixed_scaled_mm(q.A, q.CA, s.CB, q.SCA, s.SCB, q.cols,
                                                                   self._bias(dtype))
            else:
                y = torch.ops.bitsandbytes.int8_scaled_mm.default(q.CA, s.CB, q.SCA, s.SCB, bias=self._bias(dtype),
                                                                  dtype=dtype)
            out.copy_(y.view(M, s.rows))
        return out

    def _gemm(self, q: Int8Input, outs, ldc: int) -> bool:
        s = self.shard
        subA = subBT = None
        if 0 < q.J <= _INT8_FUSED_J:
            subA, subBT = (q.subA, q.subBT) if q.A is None else int8_outlier_operands(q.A, s.CB, s.SCB, q.cols)
        return int8_gemm_multi_out(q.CA, s.CB, q.SCA, s.SCB, outs, ldc, q.dtype, self._bias(q.dtype), subA, subBT)

    def outlier_rows(self, q: Int8Input) -> torch.Tensor:
        """This rank's rows [rows, J] of the dequantised outlier weight columns (J > 64: the addmm operand)."""
        s = self.shard
        return F.int8_vectorwise_dequant(s.CB[:, q.cols].contiguous(), s.SCB).to(q.dtype)

    @staticmethod
    def finish(full: torch.Tensor, q: Int8Input, subBT: torch.Tensor) -> torch.Tensor:
        """The unsharded layer's outlier step past 64 columns on the gathered [M, N] output and [N, J] weight columns:
        the same ``addmm`` on the same operands."""
        subA = q.A[:, q.cols].contiguous() if q.A is not None else q.subA
        return full.addmm(subA, subBT.t())

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _ParallelFn.apply(x, self)

    def _forward(self, x: torch.Tensor, peers=None, sp: Optional[bool] = None) -> torch.Tensor:
        """The layer's output.  ``sp`` (default: ``sequence_parallel``) chooses the mode; ``peers`` is a
        :class:`PeerInt8Input` under sequence parallelism (:meth:`sp_quantize`), a :class:`PeerGather` otherwise
        (:meth:`_output`)."""
        world, _ = _group_world_rank(self.group)
        if (self.sequence_parallel if sp is None else sp) and (world > 1 or peers is not None):
            return self._output(self.sp_quantize(x, peers), (world * x.shape[0], *x.shape[1:-1]))
        return self._output(self.quantize(x), x.shape[:-1], peers)

    def _output(self, q: Int8Input, lead, peers: Optional["PeerGather"] = None) -> torch.Tensor:
        """The layer's output from the quantised input of all M tokens (``lead``: its leading dimensions).  With
        ``peers`` the int8 GEMM epilogue stores each output element into this rank's columns of every rank's ``[M, N]``
        slot, or, past 64 outlier columns or for a shape the GEMM does not take, the NCCL route fills the slot; one
        barrier, and the slot itself is returned, whatever ``gather_output`` says."""
        s = self.shard
        M = q.CA.shape[0]
        world, _ = _group_world_rank(self.group)
        chain = q.J > _INT8_FUSED_J
        if peers is not None:
            _check_peers(peers, M, self.out_features, q.dtype, "output shape / dtype")
            local, bases, handle = peers.slot()
            if chain or not self._gemm(q, peers.dest_ptrs(bases, s.row0 * local.element_size()), peers.N):
                local.copy_(self._gathered(q, M, world, chain))
            handle.barrier(channel=0)  # every rank's stores have landed everywhere
            return local
        if world == 1:
            y = self.local_forward(q)
            if chain:
                y = self.finish(y, q, self.outlier_rows(q))
            return y.view(*lead, s.rows)
        if not self.gather_output and not chain:
            return self.local_forward(q).view(*lead, s.rows)
        full = self._gathered(q, M, world, chain)
        if not self.gather_output:
            full = full[:, s.row0:s.row0 + s.rows].contiguous()
        return full.reshape(*lead, full.shape[-1])

    def _gathered(self, q: Int8Input, M: int, world: int, chain: bool) -> torch.Tensor:
        """The ``[M, N]`` output of all ranks through NCCL: the columns all-gathered and, past 64 outlier columns, the
        unsharded layer's addmm on the all-gathered outlier weight rows."""
        full = _gather_columns(self, q, M, q.dtype, q.CA.device)
        if chain:
            subBT = torch.empty((world * self.shard.rows, q.J), device=q.CA.device, dtype=q.dtype)
            dist.all_gather_into_tensor(subBT, self.outlier_rows(q), group=self.group)
            full = self.finish(full, q, subBT)
        return full


def fused_forward_col8(layer: ColumnParallelLinear8bitLt, x: torch.Tensor, peers: PeerGather,
                      grad_peers: Optional[PeerInputGrad] = None) -> torch.Tensor:
    """``layer(x)`` with the all-gather fused into the int8 GEMM epilogue: each output element is stored into this
    rank's columns of every rank's symmetric ``[M, N]`` buffer.  Past 64 outlier columns, or for a shape the GEMM does
    not take, the local GEMM + NCCL route fills the same slot.  Returns this rank's [M, N] slot.  With ``grad_peers =
    PeerInputGrad(M, K, torch.float32)`` an input that requires grad gets its gradient (the outlier decomposition
    leaves it alone, as in the layer's own backward), and the call returns a copy of the slot, as ``fused_forward``."""
    return _fused_route("fused_forward_col8", layer, x, peers, False, grad_peers, copy_out=True)


class PeerInt8Input(_PeerSlots):
    """Two symmetric-memory slots for the gathered input of a sequence-parallel int8 column layer: ``[M*K int8 codes |
    M fp32 row statistics]`` in one buffer, so that one barrier publishes both (``K % 16 == 0`` keeps the statistics
    aligned)."""

    def __init__(self, M: int, K: int, device, group: Optional[dist.ProcessGroup] = None):
        if K % 16 != 0:
            raise ValueError(f"in_features ({K}) must be a multiple of 16")
        super().__init__((M * K + 4 * M,), torch.uint8, device, group)
        self.M, self.K = M, K

    def codes(self, local: torch.Tensor) -> torch.Tensor:
        """The int8 [M, K] codes of a slot."""
        return local[:self.M * self.K].view(torch.int8).view(self.M, self.K)

    def stats(self, local: torch.Tensor) -> torch.Tensor:
        """The fp32 [M] row statistics of a slot."""
        return local[self.M * self.K:].view(torch.float32)


def fused_forward_col8_sp(layer: ColumnParallelLinear8bitLt, x: torch.Tensor, peers: PeerInt8Input,
                          grad_peers: Optional[PeerInputGrad] = None) -> torch.Tensor:
    """The sequence-parallel ``layer(x)`` with the gather of the quantised tokens through symmetric memory: this rank
    quantises its ``[M/w, ..., K]`` tokens and copies the codes and row statistics into its rows of every rank's slot
    (``peers = PeerInt8Input(M, K)``), one barrier publishes them, and the local GEMM reads the gathered codes.  Returns
    ``[M, ..., N/w]``.  With ``grad_peers = PeerInputGrad(M, K, torch.float32)`` an input that requires grad gets the
    gradient of its tokens, reduced from the peers' partials."""
    return _fused_route("fused_forward_col8_sp", layer, x, peers, True, grad_peers)


@dataclass
class Int8Stats:
    """One rank's share of the row statistics of a row-parallel layer's input."""

    x16: torch.Tensor               # fp16 [M, K / world]: the slice as the unsharded layer quantises it
    row_stats: torch.Tensor         # fp32 [M]: absmax of the slice's entries below the threshold
    flags: Optional[torch.Tensor]   # int32 [K / world]: the slice's outlier columns (threshold > 0)


class RowParallelLinear8bitLt(_RowInputGrad, torch.nn.Module):
    """LLM.int8() ``y = x @ W^T + b`` with W's input features split across the process group: every rank returns the
    whole ``[..., N]`` output, equal to the unsharded inference ``Linear8bitLt`` output bit for bit.

    The forward pass runs in steps a single process can also drive rank by rank: :meth:`local_stats` -> a max over the
    ranks -> :meth:`local_codes` -> :meth:`partial_forward` (+ :meth:`outlier_operands`) -> an exchange ->
    :meth:`reduce`.  With ``sequence_parallel=True`` each rank returns only its tokens' rows, ``[M/w, ..., N]``."""

    def __init__(self, shard: Shard8bit, in_features: int, bias: Optional[torch.Tensor] = None,
                 group: Optional[dist.ProcessGroup] = None, input_is_parallel: bool = True, threshold: float = 0.0,
                 sequence_parallel: bool = False):
        super().__init__()
        self.shard = shard
        self.in_features = in_features
        self.out_features = shard.rows
        self.group = group
        self.input_is_parallel = input_is_parallel
        self.threshold = float(threshold)
        self.sequence_parallel = sequence_parallel
        self.bias = None if bias is None else bias.contiguous()
        self._stage = None
        self._sp_bufs = None

    @classmethod
    def from_quantized(cls, CB, SCB, bias=None, group=None, threshold: float = 0.0, input_is_parallel: bool = True,
                       sequence_parallel: bool = False):
        world, rank = _group_world_rank(group)
        return cls(slice_int8_weight_k(CB, SCB, world, rank), CB.shape[1], bias, group, input_is_parallel, threshold,
                   sequence_parallel)

    @classmethod
    def from_linear8bitlt(cls, module, group=None, input_is_parallel: bool = True, sequence_parallel: bool = False):
        CB, SCB, threshold = _state_of(module)
        return cls.from_quantized(CB, SCB, module.bias, group, threshold, input_is_parallel, sequence_parallel)

    def local_input(self, x: torch.Tensor) -> torch.Tensor:
        """This rank's ``x_r[M, K/world]``: ``x`` itself, or its slice when the layer takes the full input."""
        s = self.shard
        if self.input_is_parallel:
            if x.shape[-1] != s.K:
                raise ValueError(f"expected this rank's {s.K} input features, got {x.shape[-1]}")
            return x.reshape(-1, s.K)
        if x.shape[-1] != self.in_features:
            raise ValueError(f"expected {self.in_features} input features, got {x.shape[-1]}")
        return x.reshape(-1, self.in_features)[:, s.k0:s.k0 + s.K]

    def local_stats(self, x_r: torch.Tensor) -> Int8Stats:
        """Step 1: the slice's row absmax and outlier flags, with the unsharded quantiser's rounding."""
        _no_capture(self.threshold, "RowParallelLinear8bitLt")
        x16 = x_r.to(torch.float16).contiguous()
        row_stats, flags = int8_row_stats(x16, self.threshold)
        return Int8Stats(x16, row_stats, flags)

    def local_codes(self, st: Int8Stats, SCA: torch.Tensor) -> tuple[torch.Tensor, Optional[torch.Tensor]]:
        """Step 3: (CA_r, local outlier columns or None) from the global statistics ``SCA`` (the max over the ranks).
        The outlier columns are zeroed in CA_r for more than one row, as the unsharded quantiser does."""
        CA = int8_quant_with_stats(st.x16, SCA, self.threshold)
        if st.flags is None:
            return CA, None
        cols = torch.nonzero(st.flags).view(-1)  # data-dependent: a host synchronisation, as in the unsharded layer
        if cols.numel() and CA.shape[0] > 1:
            int8_zero_columns(CA, cols)
        return CA, cols

    def partial_forward(self, CA: torch.Tensor, outs, ldc: Optional[int] = None) -> bool:
        """Step 4: the exact int32 partial ``CA_r . CB_r^T`` to every destination in ``outs``."""
        s = self.shard
        return int8_gemm_multi_out(CA, s.CB, None, None, outs, s.rows if ldc is None else ldc, None)

    def partial_scatter(self, CA: torch.Tensor, outs, ldc: Optional[int] = None) -> bool:
        """:meth:`partial_forward` with the rows of the partial split over ``outs`` in rank order: rank s's tokens go to
        ``outs[s]`` (sequence parallelism)."""
        s = self.shard
        return int8_gemm_partial_scatter(CA, s.CB, outs, s.rows if ldc is None else ldc)

    def outlier_operands(self, x_r: torch.Tensor, cols: torch.Tensor, jpad: int):
        """(subA_r [M, jpad], subBT_r [N, jpad]): the rank's outlier columns of x and of the weight, zero-padded."""
        s = self.shard
        return int8_outlier_operands(x_r, s.CB, s.SCB, cols, jpad)

    def reduce(self, parts: torch.Tensor, SCA: torch.Tensor, dtype: torch.dtype, subA=None, subBT=None,
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Step 6: the [M, N] output from the [world, M, N] int32 partials and the global outlier operands (subA
        [M, J], subBT [N, J] in rank order, or None): the GEMM epilogue with the outlier term up to 64 columns, the
        unsharded layer's addmm beyond."""
        bias = None if self.bias is None else self.bias.to(dtype)
        J = 0 if subA is None else subA.shape[1]
        if J == 0 or J > _INT8_FUSED_J:
            y = int8_reduce_partials(parts, SCA, self.shard.SCB, dtype, bias, out=out)
            return y if J == 0 else y.addmm(subA, subBT.t())
        jpad = -(-J // 8) * 8
        pa = torch.zeros((subA.shape[0], jpad), device=subA.device, dtype=dtype)
        pb = torch.zeros((subBT.shape[0], jpad), device=subBT.device, dtype=dtype)
        pa[:, :J] = subA
        pb[:, :J] = subBT
        return int8_reduce_partials(parts, SCA, self.shard.SCB, dtype, bias, pa, pb, out=out)

    @staticmethod
    def combine_outliers(operands, counts):
        """The global (subA [M, J], subBT [N, J]) from every rank's padded operands and outlier count, in rank order
        (None when there is no outlier column)."""
        if sum(counts) == 0:
            return None, None
        subA = torch.cat([a[:, :j] for (a, _), j in zip(operands, counts)], dim=1).contiguous()
        subBT = torch.cat([b[:, :j] for (_, b), j in zip(operands, counts)], dim=1).contiguous()
        return subA, subBT

    def _outlier_counts(self, x_r, cols, world: int) -> Optional[list[int]]:
        """Every rank's outlier count in rank order, gathered through NCCL (None at threshold 0)."""
        if cols is None:
            return None
        dev = x_r.device
        counts = [int(cols.numel())]
        if world > 1:
            counts_t = torch.empty(world, device=dev, dtype=torch.int64)
            dist.all_gather_into_tensor(counts_t, torch.tensor(counts, device=dev, dtype=torch.int64), group=self.group)
            counts = counts_t.tolist()
        return counts

    def _exchange_outliers(self, x_r, cols, world: int, counts: Optional[list[int]] = None):
        """Every rank's outlier count (unless given) and operands, gathered in rank order through NCCL (None, None
        without any)."""
        if cols is None:
            return None, None
        dev = x_r.device
        if counts is None:
            counts = self._outlier_counts(x_r, cols, world)
        if sum(counts) == 0:
            return None, None
        P = max(8, -(-max(counts) // 8) * 8)
        a, b = self.outlier_operands(x_r, cols, P)
        if world == 1:
            return self.combine_outliers([(a, b)], counts)
        M = x_r.shape[0]
        every = torch.empty((world, M + self.shard.rows, P), device=dev, dtype=x_r.dtype)
        dist.all_gather_into_tensor(every.view(-1), torch.cat((a, b)).reshape(-1), group=self.group)
        return self.combine_outliers([(every[r, :M], every[r, M:]) for r in range(world)], counts)

    def _prologue(self, x: torch.Tensor):
        x_r = self.local_input(x)
        world, _ = _group_world_rank(self.group)
        st = self.local_stats(x_r)
        SCA = st.row_stats
        if world > 1:
            dist.all_reduce(SCA, op=dist.ReduceOp.MAX, group=self.group)
        CA, cols = self.local_codes(st, SCA)
        return x_r, world, SCA, CA, cols

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _ParallelFn.apply(x, self)

    def _forward(self, x: torch.Tensor, peers: Optional[PeerPartials] = None,
                 sp: Optional[bool] = None) -> torch.Tensor:
        """The layer's output.  ``sp`` (default: ``sequence_parallel``) chooses the mode (:meth:`_sp_forward`).  With
        ``peers`` the GEMM epilogue stores the int32 partial ``P_r`` into slot r of every rank's buffer, and one barrier,
        after the outlier operands have travelled through NCCL, publishes them."""
        if self.sequence_parallel if sp is None else sp:
            return self._sp_forward(x, peers)
        s = self.shard
        lead = x.shape[:-1]
        x_r, world, SCA, CA, cols = self._prologue(x)
        M = x_r.shape[0]
        if peers is None:
            parts = _gather_partials(self, CA, M, torch.int32, x.device, "the int8 GEMM")
            subA, subBT = self._exchange_outliers(x_r, cols, world)
        else:
            _check_peers(peers, M, s.rows, torch.int32, "output shape or dtype (int32 partials)")
            parts, bases, handle = peers.slot()
            if not self.partial_forward(CA, peers.dest_ptrs(bases, peers.rank * M * s.rows * 4)):
                raise RuntimeError("the int8 GEMM does not serve this shard shape")
            subA, subBT = self._exchange_outliers(x_r, cols, world)
            handle.barrier(channel=0)  # every rank's partial has landed everywhere
        return self.reduce(parts, SCA, x.dtype, subA, subBT).view(*lead, s.rows)

    def _sp_forward(self, x: torch.Tensor, peers: Optional[PeerPartials] = None) -> torch.Tensor:
        """The sequence-parallel forward: this rank's rows ``[M/w, ..., N]`` of the non-SP output.  The partials of this
        rank's tokens arrive through :func:`_sp_exchange` or, with ``peers``, from every rank's scatter GEMM into this
        rank's symmetric ``[world, M/world, N]`` slot."""
        s = self.shard
        world, rank = _group_world_rank(self.group)
        Ms = sp_rows(x, world)
        if peers is not None:
            _check_peers(peers, Ms, s.rows, torch.int32, "output shape or dtype (int32 partials)")
        x_r, world, SCA, CA, cols = self._prologue(x)
        counts = self._outlier_counts(x_r, cols, world)  # before the GEMM: every rank then takes the same route
        mine = slice(rank * Ms, (rank + 1) * Ms)
        lead = (x.shape[0] // world, *x.shape[1:-1], s.rows)
        if counts is not None and sum(counts) > _INT8_FUSED_J:
            # The slow path: an addmm on this rank's rows need not give the bits of the one on all M rows, so the
            # non-SP computation runs (all partials, full reduction, addmm) and this rank keeps its rows.
            parts = _gather_partials(self, CA, x_r.shape[0], torch.int32, x.device, "the int8 GEMM")
            subA, subBT = self._exchange_outliers(x_r, cols, world, counts)
            return self.reduce(parts, SCA, x.dtype, subA, subBT)[mine].view(lead)
        if peers is None:
            parts = _sp_exchange(self, CA, Ms, torch.int32, "the int8 GEMM")
            subA, subBT = self._exchange_outliers(x_r, cols, world, counts)
        else:
            parts, bases, handle = peers.slot()
            if not self.partial_scatter(CA, peers.scatter_ptrs(bases, peers.rank * Ms * s.rows * 4)):
                parts.copy_(_sp_exchange(self, CA, Ms, torch.int32, "the int8 GEMM"))  # the scatter GEMM refused
            subA, subBT = self._exchange_outliers(x_r, cols, world, counts)
            handle.barrier(channel=0)  # every rank's rows have landed at their owner
        return self.reduce(parts, SCA[mine], x.dtype, None if subA is None else subA[mine], subBT).view(lead)


def fused_forward_row8(layer: RowParallelLinear8bitLt, x: torch.Tensor, peers: PeerPartials,
                      grad_peers: Optional[PeerInputGrad] = None) -> torch.Tensor:
    """``layer(x)`` with the exchange of the int32 partials fused into the GEMM epilogue: ``P_r`` is stored into slot r
    of every rank's symmetric buffer, one barrier publishes them, and each rank reduces its own buffer.  The row
    statistics (a max) and the outlier operands still travel through NCCL.  With ``grad_peers`` an input that requires
    grad gets its gradient, exchanged through symmetric memory."""
    return _fused_route("fused_forward_row8", layer, x, peers, False, grad_peers)


def fused_forward_row8_sp(layer: RowParallelLinear8bitLt, x: torch.Tensor, peers: PeerPartials,
                         grad_peers: Optional[PeerInputGrad] = None) -> torch.Tensor:
    """The sequence-parallel ``layer(x)`` (this rank's tokens only) with the exchange of the int32 partials fused into
    the GEMM epilogue: the rows of ``P_r`` that belong to rank s are stored into slot r of rank s's ``[world, M/world,
    N]`` buffer (``peers = PeerPartials(M // world, N, dtype=torch.int32)``), one barrier publishes them, and each rank
    reduces its own with its rows of the statistics and outlier operands.  Past 64 outlier columns the slow path of the
    NCCL route runs instead (:meth:`RowParallelLinear8bitLt._sp_forward`).  With ``grad_peers = PeerInputGrad(M, N,
    x.dtype)`` an input that requires grad gets its gradient: the token rows of ``grad_y`` gathered through symmetric
    memory."""
    return _fused_route("fused_forward_row8_sp", layer, x, peers, True, grad_peers)
