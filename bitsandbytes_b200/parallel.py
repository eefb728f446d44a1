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

Fused exchange (``PeerGather`` + ``forward_fused``): the output lives in symmetric memory
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
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
import torch.distributed as dist

from . import functional as F
from .backends.cuda import gemm_4bit_into, gemm_4bit_multi_out, gemm_4bit_partial, reduce_partials


@dataclass
class Shard4bit:
    """The slice of a quantised [N, K] weight owned by one rank."""

    packed: torch.Tensor            # uint8 [rows*K/2]
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


class ColumnParallelLinear4bit(torch.nn.Module):
    """``y = x @ dequant(W)^T + b`` with W's output features split across the process group."""

    def __init__(self, shard: Shard4bit, out_features: int, bias: Optional[torch.Tensor] = None,
                 group: Optional[dist.ProcessGroup] = None, gather_output: bool = True):
        super().__init__()
        self.shard = shard
        self.out_features = out_features
        self.group = group
        self.gather_output = gather_output
        self.bias_shard = None if bias is None else bias[shard.row0:shard.row0 + shard.rows].contiguous()
        self._stage = None

    @classmethod
    def from_quantized(cls, packed, qs: F.QuantState, bias=None, group=None, gather_output=True):
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        rank = dist.get_rank(group) if dist.is_initialized() else 0
        return cls(slice_quantized_weight(packed, qs, world, rank), qs.shape[0], bias, group, gather_output)

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
        s = self.shard
        lead = x.shape[:-1]
        M = x.numel() // s.K
        world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        if world == 1 or not self.gather_output:
            return self.local_forward(x).view(*lead, s.rows)
        if self._stage is None or self._stage.shape[1] != M or self._stage.dtype != x.dtype:
            self._stage = torch.empty((world, M, s.rows), device=x.device, dtype=x.dtype)
        rank = dist.get_rank(self.group)
        self.local_forward(x, self._stage[rank], s.rows)
        dist.all_gather_into_tensor(self._stage.view(-1), self._stage[rank].reshape(-1), group=self.group)
        # [world, M, rows] -> [M, world*rows]
        return self._stage.permute(1, 0, 2).reshape(*lead, world * s.rows)


class PeerGather:
    """Two symmetric-memory ``[M, N]`` output slots shared by the ranks of ``group``."""

    def __init__(self, M: int, N: int, dtype: torch.dtype, device, group: Optional[dist.ProcessGroup] = None):
        import torch.distributed._symmetric_memory as symm_mem

        group = group if group is not None else dist.group.WORLD
        self.M, self.N, self.dtype = M, N, dtype
        self.bufs, self.handles = [], []
        for _ in range(2):
            t = symm_mem.empty((M, N), dtype=dtype, device=device)
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


def fused_forward(layer: "ColumnParallelLinear4bit", x: torch.Tensor, peers: PeerGather) -> torch.Tensor:
    """``layer(x)`` with the all-gather fused into the GEMM epilogue; returns this rank's [M, N] slot."""
    s = layer.shard
    M = x.numel() // s.K
    if M != peers.M or layer.out_features != peers.N or x.dtype != peers.dtype:
        raise ValueError("PeerGather was built for a different output shape / dtype")
    local, bases, handle = peers.slot()
    col_bytes = s.row0 * local.element_size()
    # own buffer first, then the peers
    order = [peers.rank] + [r for r in range(peers.world) if r != peers.rank]
    ptrs = [bases[r] + col_bytes for r in order]
    ok = gemm_4bit_multi_out(x, s.packed, (s.rows, s.K), s.absmax, s.blocksize, s.quant_type, layer.bias_shard,
                             s.absmax_8bit, s.absmax_code, s.absmax_offset, ptrs, peers.N)
    if not ok:  # shape outside the tensor-core kernel: local slice + NCCL all-gather into the same slot
        stage = torch.empty((peers.world, M, s.rows), device=x.device, dtype=x.dtype)
        layer.local_forward(x, stage[peers.rank], s.rows)
        dist.all_gather_into_tensor(stage.view(-1), stage[peers.rank].reshape(-1), group=layer.group)
        local.copy_(stage.permute(1, 0, 2).reshape(M, peers.N))
    handle.barrier(channel=0)  # every rank's stores have landed everywhere
    return local


def _ftz(t: torch.Tensor) -> torch.Tensor:
    """fp32 values below the normal range flushed to (signed) zero, as the kernels' ``mul.ftz`` does."""
    return torch.where(t.abs() < 2.0**-126, t * 0.0, t)


def nested_scales(qs: F.QuantState) -> torch.Tensor:
    """The fp32 scale of every quantisation block of a double-quantised state, computed as the kernels fetch it
    (``ScaleSrc::load_as``): ``(code2[absmax_8bit] * absmax2[block // 256])`` rounded, flushed to zero below the
    normal range, then ``+ offset`` rounded."""
    a2 = qs.state2.absmax.float()
    idx = torch.arange(qs.absmax.numel(), device=a2.device) // 256
    prod = _ftz(_ftz(qs.state2.code.float()[qs.absmax.long()]) * _ftz(a2[idx]))
    return prod + qs.offset.reshape(()).float().to(prod.device)


def slice_quantized_weight_k(packed: torch.Tensor, qs: F.QuantState, world: int, rank: int) -> Shard4bit:
    """Cut rank's input features ``W[:, k0:k1]`` out of a weight quantised once, globally (no re-quantisation).

    The slice is strided in the packed layout (``[N, K/2]`` bytes, ``[N, K/blocksize]`` absmax), so the shard is a
    repacked copy, made once at load.  Requires ``K % (world * blocksize) == 0`` and ``(K / world) % 64 == 0`` (the
    shard stays on the tensor-core kernels).  A double-quantised state's level-2 groups of 256 blocks straddle the
    shards, so the shard's scales are plain fp32 absmax computed exactly as the kernels fetch the nested ones
    (:func:`nested_scales`): the shard decodes to the same weights bit for bit."""
    N, K = qs.shape
    bs = qs.blocksize
    if world < 1 or not 0 <= rank < world:
        raise ValueError(f"rank {rank} outside a world of {world}")
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


class RowParallelLinear4bit(torch.nn.Module):
    """``y = x @ dequant(W)^T + b`` with W's input features split across the process group: every rank returns the
    whole ``[..., N]`` output, the same bits on every rank."""

    def __init__(self, shard: Shard4bit, in_features: int, bias: Optional[torch.Tensor] = None,
                 group: Optional[dist.ProcessGroup] = None, input_is_parallel: bool = True):
        super().__init__()
        self.shard = shard
        self.in_features = in_features
        self.out_features = shard.rows
        self.group = group
        self.input_is_parallel = input_is_parallel
        self.bias = None if bias is None else bias.contiguous()
        self._stage = None

    @classmethod
    def from_quantized(cls, packed, qs: F.QuantState, bias=None, group=None, input_is_parallel=True):
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        rank = dist.get_rank(group) if dist.is_initialized() else 0
        return cls(slice_quantized_weight_k(packed, qs, world, rank), qs.shape[1], bias, group, input_is_parallel)

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

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        s = self.shard
        x_r = self.local_input(x)
        lead = x_r.shape[:-1]
        M = x_r.numel() // s.K
        world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        rank = dist.get_rank(self.group) if dist.is_initialized() else 0
        if self._stage is None or self._stage.shape[:2] != (world, M) or self._stage.device != x.device:
            self._stage = torch.empty((world, M, s.rows), device=x.device, dtype=torch.float32)
        if not self.partial_forward(x_r, [self._stage[rank]]):
            raise RuntimeError("gemm_4bit_partial does not serve this shape or dtype")
        if world > 1:
            dist.all_gather_into_tensor(self._stage.view(-1), self._stage[rank].reshape(-1), group=self.group)
        return reduce_partials(self._stage, x.dtype, self.bias).view(*lead, s.rows)


class PeerPartials:
    """Two symmetric-memory ``[world, M, N]`` fp32 partial slots shared by the ranks of ``group``."""

    def __init__(self, M: int, N: int, device, group: Optional[dist.ProcessGroup] = None):
        import torch.distributed._symmetric_memory as symm_mem

        group = group if group is not None else dist.group.WORLD
        self.M, self.N = M, N
        self.bufs, self.handles = [], []
        for _ in range(2):
            t = symm_mem.empty((dist.get_world_size(group), M, N), dtype=torch.float32, device=device)
            self.handles.append(symm_mem.rendezvous(t, group))
            self.bufs.append(t)
        self.world = self.handles[0].world_size
        self.rank = self.handles[0].rank
        self.step = 0

    def slot(self):
        """(local [world, M, N] tensor, [base address of that slot on rank r for every r], handle) of the next step."""
        i = self.step & 1
        self.step += 1
        return self.bufs[i], [int(p) for p in self.handles[i].buffer_ptrs], self.handles[i]


def fused_forward_row(layer: RowParallelLinear4bit, x: torch.Tensor, peers: PeerPartials) -> torch.Tensor:
    """``layer(x)`` with the exchange of the partials fused into the GEMM epilogue: ``P_r`` is stored into slot r of
    every rank's buffer, one barrier publishes them, and each rank reduces them in rank order."""
    s = layer.shard
    x_r = layer.local_input(x)
    M = x_r.numel() // s.K
    if M != peers.M or s.rows != peers.N:
        raise ValueError("PeerPartials was built for a different output shape")
    local, bases, handle = peers.slot()
    off = peers.rank * M * s.rows * 4  # this rank's slot, in bytes
    # own buffer first, then the peers
    order = [peers.rank] + [r for r in range(peers.world) if r != peers.rank]
    if not layer.partial_forward(x_r, [bases[r] + off for r in order]):
        raise RuntimeError("gemm_4bit_partial does not serve this shape or dtype")
    handle.barrier(channel=0)  # every rank's partial has landed everywhere
    return reduce_partials(local, x.dtype, layer.bias).view(*x_r.shape[:-1], s.rows)


def reassemble_shards(shards: list[Shard4bit]) -> tuple[torch.Tensor, torch.Tensor]:
    """Inverse of slice_quantized_weight for the plain (non-nested) case: (packed, absmax)."""
    return torch.cat([s.packed for s in shards]), torch.cat([s.absmax for s in shards])
