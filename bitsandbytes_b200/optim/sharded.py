"""Optimizer state sharded over data-parallel ranks (ZeRO stage 1), with the single-GPU optimizer's results.

``ShardedOptimizer(AdamW8bit(model.parameters()))`` moves the parameters that require grad into one flat buffer per
dtype, and their gradients into a flat buffer of the same layout: tensor t starts at 256 x (the blocks of the tensors
before it), so every 256-element block of the 8-bit state is a block of one tensor, and its tail up to the block end is
padding.  The buffer holds ``w * S`` elements, ``S = ceil(B / w) * 256`` for B blocks, and rank r owns ``[r*S,
(r+1)*S)``: the pieces of the tensors inside that range, each a run of whole blocks of its tensor (plus the tensor's
last, partial block when the range holds it).  A rank keeps optimizer state for its pieces only, about 1/w of the
unsharded optimizer's bytes; whether a tensor's state is 8-bit is decided on the whole tensor (``min_8bit_size``).

``step()`` exchanges the gradients with ``all_to_all_single`` into a ``[w, S]`` buffer (rank s's slice of rank r's
gradient lands in row r on rank s), then runs one kernel per group of pieces that share their launch arguments
(``_Update.group_key``): it sums the w ranks' gradients element by element in rank order in fp32, scales the sum by
``grad_scale`` (default 1/w, the mean), rounds it once to the parameter dtype and updates the rank's pieces with the
unsharded kernels' arithmetic; an ``all_gather_into_tensor`` hands every rank the new parameters.  With one rank there
is nothing to exchange.

After k steps every rank's parameters, and ``consolidated_state_dict()``, equal bit for bit those of one unsharded
optimizer fed at each step the gradient ``T(rank-order fp32 sum * fp32(grad_scale))``, with one exception: fp32
parameters whose state is 32-bit Lion.  There the unsharded kernel contracts the decoupled weight decay and the step
into one fma in some unrolled copies of its element loop and not in others, so its own result depends on where an
element falls in the loop; the sharded parameters and state are then within a few ulp of it, and a parameter whose
``sign(beta1 * m + (1 - beta1) * g)`` argument is within rounding of zero may take the other sign.

A parameter without a gradient at ``step()`` is updated with a zero gradient, as DDP's ``find_unused_parameters``
reduces zeros; the unsharded optimizer would skip it instead.

``clip_grad_norm_(max_norm, norm_type=2.0)`` clips the global norm of the reduced gradient, which no rank holds (each
``p.grad`` is the rank's local gradient, so ``torch.nn.utils.clip_grad_norm_`` would clip by a local norm).  It does
the step's exchange early, runs a norm kernel over the rank's pieces that forms each element's gradient exactly as the
update will and accumulates in fp64, all-gathers one value per rank, and computes the norm and torch's coefficient
on the device.  ``step()`` then skips the exchange and hands the coefficient's address to the update kernels, which
apply it as the unsharded kernels apply ``gnorm_scale``: the step equals the unsharded optimizer's fed the reduced
gradient with ``gnorm_scale`` = the coefficient.

Wrapping an optimizer made with ``capturable=True`` makes ``step()`` (and ``clip_grad_norm_``) safe to capture in a CUDA
graph, with the NCCL collectives inside it: the step counters are one int32 tensor on the device, ``steps``, that
``step()`` advances for every parameter with one in-place add (on every rank, also for parameters of which the rank
holds no piece) before the update kernels read it; ``group["lr"]`` may be a one-element fp32 CUDA tensor, read by the
kernels at every launch; and ``step()`` reads nothing on the host.  The parameters must be on a CUDA device.  The exchange buffers, the clip's buffers and the
state are made by one eager ``step()`` (after an eager ``clip_grad_norm_`` if the captured region clips), which also
warms NCCL's communicator; a step that would make one of them while capturing raises.  The results are those of
``capturable=False``, bit for bit.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from ..backends.cuda import (optimizer_clip_coef, optimizer_grad_norm_peers, optimizer_update_32bit_multi_peers,
                             optimizer_update_8bit_blockwise_multi_peers)
from ..parallel import _group_world_rank
from .optimizer import _STATE_BLOCK, Optimizer2State, Optimizer8bit, _capturing, _Update, group_updates

_QUANT_KEY = Optimizer8bit._FSDP_WRAPPED_QUANT_STATE_KEY
_STATE_KEYS = ("state1", "state2", "absmax1", "absmax2")


def _graph_device(device: torch.device) -> bool:
    """Whether work on ``device`` can be captured in a CUDA graph (a CUDA device)."""
    return device.type == "cuda"


def _blocks(n: int) -> int:
    return -(-n // _STATE_BLOCK)


def partition(numels, world: int):
    """The layout of one flat buffer: (starts, S, pieces), pieces[r] = [(tensor index, offset in the tensor, numel)] of
    rank r, in tensor order."""
    starts, B = [], 0
    for n in numels:
        starts.append(B * _STATE_BLOCK)
        B += _blocks(n)
    S = -(-B // world) * _STATE_BLOCK
    pieces = []
    for r in range(world):
        lo, hi, mine = r * S, (r + 1) * S, []
        for t, (s, n) in enumerate(zip(starts, numels)):
            a, b = max(lo, s), min(hi, s + n)
            if a < b:
                mine.append((t, a - s, b - a))
        pieces.append(mine)
    return starts, S, pieces


class _PieceUpdate(_Update):
    """A piece's launch arguments: p, its view of the local flat parameters; g, of the flat gradient."""

    __slots__ = ("flat", "g")


class _Flat:
    """The parameters of one dtype: flat parameter and gradient buffers, the layout, this rank's pieces."""

    def __init__(self, params, dtype, device, world: int, rank: int):
        self.params, self.dtype = params, dtype
        self.numels = [p.numel() for p in params]
        self.starts, self.S, pieces = partition(self.numels, world)
        self.pieces = pieces[rank]
        n = world * self.S
        self.param = torch.zeros(n, dtype=dtype, device=device)
        self.grad = torch.zeros(n, dtype=dtype, device=device)
        self.recv = None  # the [w, S] gradient exchange buffer, made at the first step


class ShardedOptimizer(torch.optim.Optimizer):
    """Shard a bnb optimizer's state over the data-parallel ranks of ``group`` (see the module documentation).

    ``optimizer``: an 8-bit / 32-bit / mixed Adam, AdamW, SGD (momentum), RMSprop, Adagrad or Lion of ``bnb.optim``
    that has taken no step.  Its ``param_groups`` are this object's, so learning-rate schedulers work on either.
    ``grad_scale``: the factor of the summed gradient, 1/w (the mean) by default.  The model is not wrapped: run
    ``loss.backward(); opt.step(); opt.zero_grad()`` on every rank.  An optimizer made with ``capturable=True`` gives a
    step that can be captured in a CUDA graph (see the module documentation)."""

    def __init__(self, optimizer, group=None, grad_scale: Optional[float] = None):
        if not isinstance(optimizer, Optimizer8bit):
            raise ValueError(f"ShardedOptimizer wraps a bitsandbytes_b200 optimizer, got {type(optimizer).__name__}")
        if optimizer.is_paged:
            raise ValueError("ShardedOptimizer does not support paged optimizer state")
        if optimizer.optimizer_name == "ademamix":
            raise ValueError("ShardedOptimizer does not support AdEMAMix: its kernels address the third state "
                             "relative to the whole tensor")
        if any(len(s) for s in optimizer.state.values()):
            raise ValueError("ShardedOptimizer wraps an optimizer that has taken no step: this one already has state")
        # (torch's constructor for the hooks and the type learning-rate schedulers check; the groups are then shared)
        super().__init__([dict(g) for g in optimizer.param_groups], optimizer.defaults)
        self.optimizer, self.group = optimizer, group
        self.param_groups, self.defaults = optimizer.param_groups, optimizer.defaults
        optimizer.check_overrides()
        self.world, self.rank = _group_world_rank(group)
        self.grad_scale = 1.0 / self.world if grad_scale is None else float(grad_scale)
        # (gindex, pindex, p, config) of every parameter that requires grad, in the optimizer's order
        self.entries = []
        for gi, g in enumerate(optimizer.param_groups):
            for pi, p in enumerate(g["params"]):
                if p.requires_grad:
                    config = optimizer.get_config(gi, pi, g)
                    if config["max_unorm"] > 0.0:
                        raise ValueError("ShardedOptimizer does not support max_unorm > 0 (LAMB, LARS): the trust "
                                         "ratio needs the whole tensor's norm")
                    self.entries.append((gi, pi, p, config))
        devices = {p.device for _, _, p, _ in self.entries}
        if len(devices) > 1:
            raise ValueError(f"ShardedOptimizer needs every parameter on one device, got {sorted(map(str, devices))}")
        self.device = devices.pop() if devices else torch.device("cuda", torch.cuda.current_device())
        if optimizer.capturable and not _graph_device(self.device):
            raise ValueError(f"ShardedOptimizer with capturable=True needs its parameters on a CUDA device, got "
                             f"{self.device}: the step counters live there and the step is captured in a CUDA graph")
        by_dtype = {}
        for i, (_, _, p, _) in enumerate(self.entries):
            by_dtype.setdefault(p.dtype, []).append(i)
        self.capturable = optimizer.capturable
        self.flats = []
        if self.capturable:  # one device counter per parameter; _counters[e] is entry e's one-element view
            self.steps = torch.zeros(len(self.entries), dtype=torch.int32, device=self.device)
            self._counters = list(self.steps.split(1))
        else:
            self.steps = [0] * len(self.entries)
        self._clip = None  # (gradient sources, coefficient) from clip_grad_norm_ until the step that uses them
        self._norm_bufs = None  # capturable: the clip's accumulator, per-rank values and (norm, coefficient)
        for dtype, idx in by_dtype.items():
            flat = _Flat([self.entries[i][2] for i in idx], dtype, self.device, self.world, self.rank)
            flat.index = idx
            self._bind(flat)
            self.flats.append(flat)
        self._make_state()

    # ---- construction
    def _bind(self, flat: _Flat) -> None:
        """Parameters into the flat buffer (rank 0's values on every rank), gradients as views of the flat gradient."""
        with torch.no_grad():
            for p, s, n in zip(flat.params, flat.starts, flat.numels):
                flat.param[s:s + n].copy_(p.data.reshape(-1))
            if self.world > 1:
                src = dist.get_global_rank(self.group, 0) if self.group is not None else 0
                dist.broadcast(flat.param, src=src, group=self.group)
        flat.views = []
        for p, s, n in zip(flat.params, flat.starts, flat.numels):
            if p.grad is not None:
                flat.grad[s:s + n].copy_(p.grad.reshape(-1))
            p.data = flat.param[s:s + n].view_as(p)
            p.grad = flat.grad[s:s + n].view_as(p)
            flat.views.append(p.grad)

    def _make_state(self) -> None:
        """State of this rank's pieces: 8-bit or 32-bit as the whole tensor's would be."""
        opt = self.optimizer
        two = isinstance(opt, Optimizer2State)
        self.pieces = []  # (flat, entry index, first flat element, numel, state)
        for flat in self.flats:
            for t, off, n in flat.pieces:
                e = flat.index[t]
                _, _, p, config = self.entries[e]
                dtype = opt._state_dtype(config, p)
                st = {"state1": torch.zeros(n, dtype=dtype, device=self.device)}
                if two:
                    st["state2"] = torch.zeros(n, dtype=dtype, device=self.device)
                if dtype == torch.uint8:
                    st["qmap1"] = opt._qmap("dynamic", self.device)
                    st["absmax1"] = torch.zeros(_blocks(n), dtype=torch.float32, device=self.device)
                    if two:
                        st["qmap2"] = opt._qmap("udynamic", self.device)
                        st["absmax2"] = torch.zeros(_blocks(n), dtype=torch.float32, device=self.device)
                self.pieces.append((flat, e, flat.starts[t] + off, n, st))

    # ---- the training loop
    def zero_grad(self, set_to_none: bool = True) -> None:
        """Zero the flat gradients; every ``p.grad`` stays (or becomes again) its view of the flat gradient."""
        for flat in self.flats:
            flat.grad.zero_()
            for p, v in zip(flat.params, flat.views):
                p.grad = v

    def _gather_grads(self) -> None:
        """A ``p.grad`` that is not its view (None, or rebound by the user) goes into its slot: zeros for None."""
        with torch.no_grad():
            for flat in self.flats:
                for p, v, s, n in zip(flat.params, flat.views, flat.starts, flat.numels):
                    if p.grad is v:
                        continue
                    if p.grad is None:
                        flat.grad[s:s + n].zero_()
                    else:
                        flat.grad[s:s + n].copy_(p.grad.reshape(-1))
                    p.grad = v

    def _updates(self):
        """The launch arguments of this rank's pieces, grouped as the unsharded optimizer groups its tensors."""
        opt, two = self.optimizer, isinstance(self.optimizer, Optimizer2State)
        updates = []
        for flat, e, s, n, st in self.pieces:
            gi, pi, _, _ = self.entries[e]
            config = opt.get_config(gi, pi, self.param_groups[gi])  # (read at every step: lr schedules)
            st["step"] = self._counters[e] if self.capturable else self.steps[e]
            betas = config["betas"]
            beta3 = betas[2] if two and len(betas) >= 3 else 0.0
            u = _PieceUpdate(opt.optimizer_name, flat.param[s:s + n], st, config, betas[0], betas[1], beta3,
                        config.get("alpha", 0.0) if two else 0.0)
            u.flat, u.g = flat, flat.grad[s:s + n]
            updates.append(u)
        return group_updates(updates)

    def _launch(self, batch, srcs, dsts, coef=None) -> None:
        u, st = batch[0], batch[0].state
        flat = u.flat
        g, p = [b.g for b in batch], [b.p for b in batch]
        s1 = [b.state["state1"] for b in batch]
        s2 = [b.state["state2"] for b in batch] if "state2" in st else None
        steps = [b.state["step"] for b in batch]
        scaled = {} if coef is None else {"gnorm_scale_dev": coef}  # (no clip: the unscaled entries, as before)
        if st["state1"].dtype == torch.float32:
            optimizer_update_32bit_multi_peers(u.name, g, p, s1, s2, u.beta1, u.beta2, u.beta3, u.alpha, u.eps,
                                               u.weight_decay, steps, u.lr, srcs, dsts, flat.grad, flat.param,
                                               self.grad_scale, skip_zeros=u.skip_zeros, **scaled)
        else:
            a1 = [b.state["absmax1"] for b in batch]
            a2 = [b.state["absmax2"] for b in batch] if s2 is not None else None
            optimizer_update_8bit_blockwise_multi_peers(u.name, g, p, s1, s2, u.beta1, u.beta2, u.beta3, u.alpha,
                                                        u.eps, steps, u.lr, st["qmap1"], st.get("qmap2"), a1, a2,
                                                        u.weight_decay, srcs, dsts, flat.grad, flat.param,
                                                        self.grad_scale, skip_zeros=u.skip_zeros, **scaled)

    @torch.no_grad()
    def clip_grad_norm_(self, max_norm: float, norm_type: float = 2.0, error_if_nonfinite: bool = False):
        """Clip the global norm of the reduced gradient to ``max_norm``, as FSDP's method of the same name; call it
        between ``backward()`` and ``step()``.  Returns the total norm, a 0-dim fp32 CUDA tensor with the same bits on
        every rank.

        The gradients are exchanged now (the ``all_to_all_single`` of the step, which ``step()`` then skips).  One
        kernel per flat buffer forms this rank's elements of the reduced gradient exactly as the update will, and
        accumulates their squares (norm_type 2) or max |g| (inf) in fp64; an ``all_gather_into_tensor`` of one value per
        rank and a one-thread kernel give the norm, ``sqrt`` of the rank-order sum rounded once to fp32, and the
        coefficient ``(max_norm / (total_norm + 1e-6)).clamp(max=1.0)``, torch's bits on that norm.  The coefficient
        stays in device memory; ``step()`` hands its address to the update kernels, which apply it as the unsharded
        kernels apply ``gnorm_scale``.  Nothing is read on the host, unless ``error_if_nonfinite``: then a non-finite
        norm raises ``RuntimeError`` (one synchronisation), and ``step()`` would exchange the gradients afresh.

        Capturable: the call can be captured in a CUDA graph, except with ``error_if_nonfinite`` (a host read), which
        raises while capturing.  Its buffers are made by the first, eager call and reused, so the returned norm is
        overwritten by the next call (or replay).

        Unlike ``torch.nn.utils.clip_grad_norm_``: ``p.grad`` is not modified (the local gradients are not the reduced
        ones; the coefficient is applied inside the update); the norm is computed in fp64 from the reduced gradient and
        returned in fp32, where torch computes per-tensor norms in the gradient's dtype.  Calling torch's function on a
        sharded model's parameters clips each rank's local gradients by a local norm, which is not this step.

        ``step()`` uses the gradients as they were here.  A NaN or Inf gradient gives a NaN or Inf norm and torch's
        coefficient for it (NaN or 0), which the update then applies."""
        if not isinstance(norm_type, (int, float)) or float(norm_type) not in (2.0, float("inf")):
            raise ValueError(f"clip_grad_norm_: norm_type must be 2 or inf, got {norm_type!r}")
        if self._clip is not None:
            raise RuntimeError("clip_grad_norm_ was already called for this step: call step() first")
        capturing = _capturing()
        if capturing and error_if_nonfinite:
            raise RuntimeError("clip_grad_norm_(error_if_nonfinite=True) is being captured in a CUDA graph: the check "
                               "reads the norm on the host.  Capture it with error_if_nonfinite=False.")
        if self.capturable and self._norm_bufs is None:
            if capturing:
                raise RuntimeError(f"{type(self).__name__}.clip_grad_norm_() would create its buffers while a CUDA "
                                   "graph is being captured: run one eager clip_grad_norm_() and step() before "
                                   "capturing")
            self._norm_bufs = self._new_norm_bufs()
        self._gather_grads()
        srcs = self._exchange_grads()
        acc, every, out = self._norm_bufs if self.capturable else self._new_norm_bufs()
        acc.zero_()
        for f in self.flats:
            g = [f.grad[s:s + n] for flat, _, s, n, _ in self.pieces if flat is f]
            optimizer_grad_norm_peers(g, srcs[id(f)], f.grad, self.grad_scale, norm_type, acc)
        if self.world > 1:
            dist.all_gather_into_tensor(every, acc, group=self.group)
        optimizer_clip_coef(every, norm_type, max_norm, out)
        total = out[0]
        if error_if_nonfinite and not torch.isfinite(total).item():
            raise RuntimeError(f"The total norm of order {float(norm_type)} for gradients from `parameters` is "
                               "non-finite, so it cannot be clipped. To disable this error and scale the gradients "
                               "by the non-finite norm anyway, set `error_if_nonfinite=False`")
        self._clip = (srcs, out[1:])
        return total

    def _new_norm_bufs(self):
        """(fp64 accumulator, the ranks' fp64 values: the accumulator itself at one rank, fp32 (norm, coefficient)).
        The accumulator is zeroed by each clip_grad_norm_."""
        acc = torch.empty(1, dtype=torch.float64, device=self.device)
        every = torch.empty(self.world, dtype=torch.float64, device=self.device) if self.world > 1 else acc
        return acc, every, torch.empty(2, dtype=torch.float32, device=self.device)

    @torch.no_grad()
    def step(self, closure=None):
        if _capturing() and not self.capturable:
            raise RuntimeError(f"{type(self).__name__}.step() is being captured in a CUDA graph, but the optimizer was "
                               "constructed with capturable=False: every replay would repeat this step's step number "
                               "and learning rate.  Construct it with capturable=True.")
        if closure is not None and self._clip is not None:
            raise RuntimeError("step(closure) after clip_grad_norm_: the closure would recompute gradients that were "
                               "already exchanged and clipped")
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        clip, self._clip = self._clip, None
        if clip is None:  # (unless clip_grad_norm_ exchanged them: clip = (sources, coefficient))
            self._gather_grads()
            clip = (self._exchange_grads(), None)
        if self.capturable:
            self.steps.add_(1)
        else:
            self.steps = [k + 1 for k in self.steps]
        self._exchange(self._updates(), *clip)
        return loss

    def _exchange_grads(self):
        """Gradients in by all-to-all: id(flat) -> the w gradient source addresses of this rank's pieces."""
        srcs = {}
        for f in self.flats:
            if self.world == 1:  # nothing to exchange: the local gradient is the only source
                srcs[id(f)] = [f.grad.data_ptr()]
                continue
            if f.recv is None:
                if _capturing():
                    raise RuntimeError(f"{type(self).__name__} would create its gradient exchange buffer while a CUDA "
                                       "graph is being captured: run one eager step() before capturing")
                f.recv = torch.empty_like(f.grad)
            dist.all_to_all_single(f.recv, f.grad, group=self.group)
            es, s0 = f.grad.element_size(), self.rank * f.S
            srcs[id(f)] = [f.recv.data_ptr() + (r * f.S - s0) * es for r in range(self.world)]
        return srcs

    def _exchange(self, batches, srcs, coef) -> None:
        """One launch per batch of pieces on the exchanged gradients (srcs, as from _exchange_grads; coef: the clip
        coefficient or None), parameters out by all-gather."""
        for batch in batches:
            f = batch[0].flat
            self._launch(batch, srcs[id(f)], [f.param.data_ptr()], coef)
        if self.world == 1:
            return
        for f in self.flats:
            s0 = self.rank * f.S
            dist.all_gather_into_tensor(f.param, f.param[s0:s0 + f.S], group=self.group)

    # ---- checkpoints
    def _param_ids(self):
        """id(p) -> index in the optimizer's state dict (torch numbers the parameters across the groups)."""
        ids, k = {}, 0
        for g in self.param_groups:
            for p in g["params"]:
                ids[id(p)] = k
                k += 1
        return ids

    def _host_steps(self) -> list:
        """The steps as ints (capturable: read from the device counters, refused while capturing a graph)."""
        if not self.capturable:
            return self.steps
        if _capturing():
            raise RuntimeError(f"{type(self).__name__}: a state dict is being taken while a CUDA graph is being "
                               "captured: it reads the step counters on the host")
        return self.steps.tolist()

    def state_dict(self):
        """This rank's shard: every piece's state with its tensor, offset and size, and the partition it came from."""
        steps = self._host_steps()
        ids = self._param_ids()
        pieces = []
        for flat, e, s, n, st in self.pieces:
            pieces.append({"param": ids[id(self.entries[e][2])], "offset": s - flat.starts[flat.index.index(e)], "numel": n,
                           "state": {k: v for k, v in st.items() if k in _STATE_KEYS}})
        sd = self.optimizer.state_dict()
        return {"sharded": {"world": self.world, "rank": self.rank,
                            "numels": [[f.numels[t] for t in range(len(f.numels))] for f in self.flats]},
                "pieces": pieces, "steps": {ids[id(p)]: steps[i] for i, (_, _, p, _) in enumerate(self.entries)},
                "param_groups": sd["param_groups"]}

    def consolidated_state_dict(self, to: int = 0):
        """The unsharded optimizer's ``state_dict()``, with its tensors on the CPU, on group rank ``to``; None on the
        other ranks.  Only rank ``to`` receives the other shards, so no GPU holds the whole state."""
        mine = self.state_dict()
        steps = mine["steps"]
        local = [{"param": q["param"], "offset": q["offset"], "numel": q["numel"],
                  "state": {k: v.cpu() for k, v in q["state"].items()}} for q in mine["pieces"]]
        if self.world > 1:
            every = [None] * self.world if self.rank == to else None
            dst = dist.get_global_rank(self.group, to) if self.group is not None else to
            dist.gather_object(local, every, dst=dst, group=self.group)
            if self.rank != to:
                return None
        else:
            every = [local]
        by_param = {}
        for shard in every:
            for q in shard:
                by_param.setdefault(q["param"], []).append(q)
        ids = self._param_ids()
        opt = self.optimizer
        state = {}
        for i, (_, _, p, config) in enumerate(self.entries):
            k = ids[id(p)]
            parts = sorted(by_param.get(k, []), key=lambda q: q["offset"])
            wrapped = {}
            for key in _STATE_KEYS:
                if parts and key in parts[0]["state"]:
                    full = torch.cat([q["state"][key] for q in parts])
                    wrapped[key] = full.view(p.shape) if key.startswith("state") else full
            if not parts:  # an empty tensor: the unsharded optimizer's zero-size state
                dtype = opt._state_dtype(config, p)
                wrapped["state1"] = torch.zeros(p.shape, dtype=dtype)
                if isinstance(opt, Optimizer2State):
                    wrapped["state2"] = torch.zeros(p.shape, dtype=dtype)
                if dtype == torch.uint8:
                    wrapped["absmax1"] = torch.zeros(0)
                    if isinstance(opt, Optimizer2State):
                        wrapped["absmax2"] = torch.zeros(0)
            if wrapped["state1"].dtype == torch.uint8:
                wrapped["qmap1"] = opt._qmap("dynamic", self.device).cpu()
                if "state2" in wrapped:
                    wrapped["qmap2"] = opt._qmap("udynamic", self.device).cpu()
            state[k] = {"step": steps[k], _QUANT_KEY: wrapped}
        return {"state": state, "param_groups": mine["param_groups"]}

    def load_state_dict(self, state_dict) -> None:
        """Load this optimizer's own shard (same world, rank and parameters), or an unsharded optimizer's state dict
        (``consolidated_state_dict()`` or a plain optimizer's), of which every rank takes its blocks: a checkpoint taken
        at one world size loads at another through the consolidated form."""
        groups = state_dict["param_groups"]
        if len(groups) != len(self.param_groups) or any(len(g["params"]) != len(s["params"])
                                                        for g, s in zip(self.param_groups, groups)):
            raise ValueError("loaded state dict does not match the optimizer's parameter groups")
        ids = self._param_ids()
        if "sharded" in state_dict:
            mine = self.state_dict()
            if state_dict["sharded"] != mine["sharded"] or [(q["param"], q["offset"], q["numel"])
                                                            for q in state_dict["pieces"]] != \
                    [(q["param"], q["offset"], q["numel"]) for q in mine["pieces"]]:
                raise ValueError("this shard was saved with another partition (world, rank or parameters): load the "
                                 "consolidated_state_dict() instead")
            for (_, _, _, _, st), q in zip(self.pieces, state_dict["pieces"]):
                for key, v in q["state"].items():
                    self._load(st, key, v)
            steps = state_dict["steps"]
        else:
            full = state_dict["state"]
            for flat, e, s, n, st in self.pieces:
                k = ids[id(self.entries[e][2])]
                off = s - flat.starts[flat.index.index(e)]
                if k not in full:
                    raise ValueError(f"loaded state dict has no state for parameter {k}")
                src = dict(full[k])
                src.update(src.pop(_QUANT_KEY, {}))
                for key in _STATE_KEYS:
                    if key not in src:
                        continue
                    v = src[key].reshape(-1)
                    part = v[off:off + n] if key.startswith("state") else v[off // _STATE_BLOCK:
                                                                              off // _STATE_BLOCK + _blocks(n)]
                    if key in st and part.dtype != st[key].dtype:
                        raise ValueError(f"loaded state of parameter {k} is {part.dtype}, this optimizer keeps "
                                         f"{st[key].dtype}")
                    self._load(st, key, part)
            steps = {k: int(v["step"]) for k, v in full.items()}
        steps = [int(steps.get(ids[id(p)], 0)) for _, _, p, _ in self.entries]
        if self.capturable:  # in place, as the state: a graph captured before the load continues from it
            self.steps.copy_(torch.tensor(steps, dtype=torch.int32))
        else:
            self.steps = steps
        for g, s in zip(self.param_groups, groups):
            g.update({k: v for k, v in s.items() if k != "params"})

    def _load(self, st, key, v) -> None:
        """One state tensor of a piece: a copy on the device; capturable, written into the tensor a graph captured."""
        if self.capturable and key in st and st[key].shape == v.shape and st[key].dtype == v.dtype:
            st[key].copy_(v)
        else:
            st[key] = v.to(self.device, copy=True)
