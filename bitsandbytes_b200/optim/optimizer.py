"""Optimizer base classes with 32-bit or blockwise 8-bit state (SURVEY.md section 8 row f-4).

API mirror of the reference's ``bitsandbytes/optim/optimizer.py`` (GlobalOptimManager :26-115, Optimizer8bit
:117-401, Optimizer2State :403-590, Optimizer1State :593-756): same constructor arguments, state-dict keys
(``state1``, ``state2``, ``qmap1``, ``qmap2``, ``absmax1``, ``absmax2``, ``unorm_vec``, ``step``), per-parameter
overrides and the ``min_8bit_size`` rule, so that a checkpoint written by either implementation loads in the
other.  Unlike the reference, ``step()`` updates all parameters that share their launch arguments in one native call
(``functional.optimizer_update_32bit_multi`` / ``optimizer_update_8bit_blockwise_multi``, kernels in
``csrc/optim.cu``), with the results of one call per parameter bit for bit; ``update_step`` still updates one
parameter.

``capturable=True`` makes ``step()`` safe to capture in a CUDA graph: every ``state["step"]`` is an int32 counter on the
parameter's device that the kernels advance, ``group["lr"]`` may be a one-element fp32 CUDA tensor read at every launch,
and ``step()`` reads nothing on the host.  The results are those of ``capturable=False``, bit for bit.
"""
from __future__ import annotations

from collections import abc as container_abcs, defaultdict
from copy import deepcopy
from itertools import chain
from typing import Optional

import torch

from .. import functional as F

_STATE_BLOCK = 256  # elements per absmax of the 8-bit state (reference optimizer.py:527, csrc/ops.cu:154-157)


class MockArgs:
    def __init__(self, initial_data):
        for key, value in initial_data.items():
            setattr(self, key, value)


class _Update:
    """One parameter's launch arguments: what ``update_step`` computes (advancing ``state["step"]``) before it launches."""

    __slots__ = ("name", "p", "state", "beta1", "beta2", "beta3", "alpha", "eps", "weight_decay", "lr", "skip_zeros",
                 "max_unorm")

    def __init__(self, name, p, state, config, beta1, beta2, beta3, alpha):
        self.name, self.p, self.state = name, p, state
        self.beta1, self.beta2, self.beta3, self.alpha = beta1, beta2, beta3, alpha
        self.eps, self.weight_decay, self.lr = config["eps"], config["weight_decay"], config["lr"]
        self.skip_zeros, self.max_unorm = config["skip_zeros"], config["max_unorm"]

    def per_parameter(self) -> bool:
        """32-bit state with a trust ratio (LAMB / LARS) needs the parameter's norm and a norm pre-pass: one launch each."""
        return self.max_unorm > 0.0 and self.state["state1"].dtype == torch.float32

    def group_key(self):
        """Parameters with equal keys share every per-launch argument of the multi-tensor call.  A tensor lr is keyed
        by identity: the kernel reads it, whatever its value."""
        st = self.state
        eight = st["state1"].dtype == torch.uint8
        lr = ("tensor", id(self.lr)) if isinstance(self.lr, torch.Tensor) else self.lr
        return (self.p.device, self.p.dtype, eight, self.name, self.beta1, self.beta2, self.beta3, self.alpha, self.eps,
                self.weight_decay, lr, self.skip_zeros,
                id(st["qmap1"]) if eight else None, id(st.get("qmap2")) if eight else None)


def group_updates(updates):
    """The multi-tensor calls of one step: the updates grouped by launch arguments, in order of first appearance.  (A
    group longer than a launch's descriptor capacity is split by the backend.)"""
    groups = {}
    for u in updates:
        groups.setdefault(u.group_key(), []).append(u)
    return list(groups.values())


def _capturing() -> bool:
    """Whether the current CUDA stream is capturing a graph (impossible before CUDA is initialised)."""
    return torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing()


_NO_TRUST_RATIO = ("capturable=True does not support 32-bit state with max_unorm > 0 (LAMB / LARS): the trust ratio "
                   "needs the parameter's norm on the host at every step")
_NO_SCHEDULES = ("capturable=True does not support AdEMAMix's t_alpha / t_beta3: their schedules are computed on the "
                 "host from the step")


class GlobalOptimManager:
    """Per-parameter hyper-parameter overrides (e.g. keep an embedding's state in 32 bits)."""

    _instance = None

    def __init__(self):
        raise RuntimeError("Call get_instance() instead")

    def initialize(self):
        self.pid2config = {}
        self.index2config = {}
        self.optimizer = None
        self.uses_config_override = False
        self.module_weight_config_triple = []

    @classmethod
    def get_instance(cls):
        if cls._instance is None:
            cls._instance = cls.__new__(cls)
            cls._instance.initialize()
        return cls._instance

    def register_parameters(self, params):
        groups = list(params)
        if groups and not isinstance(groups[0], dict):
            groups = [{"params": groups}]
        for gindex, group in enumerate(groups):
            for pindex, p in enumerate(group["params"]):
                if id(p) in self.pid2config:
                    self.index2config[(gindex, pindex)] = self.pid2config[id(p)]

    def override_config(self, parameters, key=None, value=None, key_value_dict=None):
        self.uses_config_override = True
        if isinstance(parameters, (torch.nn.Parameter, torch.Tensor)):
            parameters = [parameters]
        if key is not None and value is not None:
            assert key_value_dict is None
            key_value_dict = {key: value}
        if key_value_dict is not None:
            for p in parameters:
                self.pid2config.setdefault(id(p), {}).update(key_value_dict)

    def register_module_override(self, module, param_name, config):
        self.module_weight_config_triple.append((module, param_name, config))


class Optimizer8bit(torch.optim.Optimizer):
    _FSDP_WRAPPED_QUANT_STATE_KEY = "__bnb_optimizer_quant_state__"

    def __init__(self, params, defaults, optim_bits=32, is_paged=False, capturable=False):
        super().__init__(params, defaults)
        self.initialized = False
        self.name2qmap = {}
        self.is_paged = is_paged
        self.capturable = bool(capturable)
        self.page_mng = F.GlobalPageManager.get_instance()
        self.mng = GlobalOptimManager.get_instance()
        # tensors of the state that must keep their dtype when a state dict is loaded
        self.non_castable_tensor_keys = {"qmap1", "qmap2", "max1", "max2", "new_max1", "new_max2", "state1", "state2",
                                         "gnorm_vec", "absmax1", "absmax2", "unorm_vec"}
        if optim_bits == 8:
            self.fill_qmap()

    def fill_qmap(self):
        self.name2qmap["dynamic"] = F.create_dynamic_map(signed=True)
        self.name2qmap["udynamic"] = F.create_dynamic_map(signed=False)

    # ---- state dict: the quantisation tensors travel under one wrapped key so that FSDP's flattening (which
    # expects every state tensor to have the parameter's shape) leaves them alone (reference optimizer.py:161-187)
    def state_dict(self):
        sd = super().state_dict()
        packed = {}
        for key, param_state in sd["state"].items():  # (torch hands out the live per-parameter dicts: copy, don't pop)
            plain = {k: v for k, v in param_state.items() if k not in self.non_castable_tensor_keys}
            if isinstance(plain.get("step"), torch.Tensor):  # a capturable optimizer's counter: saved as an int
                plain["step"] = int(plain["step"].item())
            wrapped = {k: v for k, v in param_state.items() if k in self.non_castable_tensor_keys}
            if wrapped:
                plain[self._FSDP_WRAPPED_QUANT_STATE_KEY] = wrapped
            packed[key] = plain
        sd["state"] = packed
        return sd

    def __setstate__(self, state):
        super().__setstate__(state)

    def load_state_dict(self, state_dict, move_to_device=True):
        state_dict = deepcopy(state_dict)
        for param_state in state_dict["state"].values():
            wrapped = param_state.pop(self._FSDP_WRAPPED_QUANT_STATE_KEY, None)
            if wrapped is not None:
                param_state.update(wrapped)
        groups = self.param_groups
        saved_groups = state_dict["param_groups"]
        if len(groups) != len(saved_groups):
            raise ValueError("loaded state dict has a different number of parameter groups")
        if any(len(g["params"]) != len(s["params"]) for g, s in zip(groups, saved_groups)):
            raise ValueError("loaded state dict contains a parameter group that doesn't match the size of optimizer's group")
        id_map = dict(zip(chain.from_iterable(g["params"] for g in saved_groups),
                          chain.from_iterable(g["params"] for g in groups)))

        def cast(param, value):
            if isinstance(value, torch.Tensor):
                # floating-point state follows the parameter's dtype; the quantisation tensors never do
                if param.is_floating_point() and value.dtype != torch.uint8:
                    value = value.to(param.dtype)
                return value
            if isinstance(value, dict):
                for k, v in value.items():
                    if k in self.non_castable_tensor_keys:
                        # (also a state that was paged when it was saved: it is reloaded as a plain device tensor)
                        if move_to_device and isinstance(v, torch.Tensor):
                            value[k] = v.to(param.device)
                    else:
                        value[k] = cast(param, v)
                return value
            if isinstance(value, container_abcs.Iterable) and not isinstance(value, str):
                return type(value)(cast(param, v) for v in value)
            return value

        state = defaultdict(dict)
        for k, v in state_dict["state"].items():
            if k in id_map:
                state[id_map[k]] = cast(id_map[k], v)
            else:
                state[k] = v

        def update_group(group, new_group):
            new_group["params"] = group["params"]
            return new_group

        self.__setstate__({"state": state, "param_groups": [update_group(g, ng) for g, ng in zip(groups, saved_groups)]})
        self._share_qmaps()
        if self.capturable:
            for p, st in self.state.items():
                if "step" in st and isinstance(p, torch.Tensor):
                    st["step"] = self._initial_step(p, int(st["step"]))

    def _share_qmaps(self):
        """A loaded state holds its own copy of the code books in every parameter: point the copies equal to this
        optimizer's code books back at them, so that the parameters share one multi-tensor call again."""
        for st in self.state.values():
            for key, name in (("qmap1", "dynamic"), ("qmap2", "udynamic")):
                q = st.get(key)
                if isinstance(q, torch.Tensor) and q.is_cuda:
                    shared = self._qmap(name, q.device)
                    if q is not shared and torch.equal(q, shared):
                        st[key] = shared

    def to_gpu(self):
        for group in self.param_groups:
            for p in group["params"]:
                if p in self.state:
                    values = self.state[p]
                    for k, v in values.items():
                        if isinstance(v, torch.Tensor) and not getattr(v, "is_paged", False):
                            self.state[p][k] = v.to(p.device)

    def check_overrides(self):
        for module, attr, config in self.mng.module_weight_config_triple:
            pmodule = getattr(module, attr)
            assert isinstance(pmodule, (torch.Tensor, torch.nn.Parameter))
            for gindex, group in enumerate(self.param_groups):
                hit = [pindex for pindex, p in enumerate(group["params"]) if p is pmodule]
                if hit:
                    self.mng.pid2config[id(pmodule)] = config
                    self.mng.index2config[(gindex, hit[0])] = config
                    break

    @torch.no_grad()
    def step(self, closure=None):
        capturing = _capturing()
        if capturing and not self.capturable:
            raise RuntimeError(f"{type(self).__name__}.step() is being captured in a CUDA graph, but the optimizer was "
                               "constructed with capturable=False: every replay would repeat this step's step number "
                               "and learning rate.  Construct it with capturable=True.")
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if not self.initialized:
            self.check_overrides()
            self.to_gpu()
            self.initialized = True
        multi = self._steps_in_groups()
        last = None
        updates = []
        for gindex, group in enumerate(self.param_groups):
            for pindex, p in enumerate(group["params"]):
                if p.grad is None:
                    continue
                if len(self.state[p]) == 0:
                    if capturing:
                        raise RuntimeError(f"{type(self).__name__}.step() would create optimizer state while a CUDA "
                                           "graph is being captured: run one eager step() before capturing")
                    self.init_state(group, p, gindex, pindex)
                self.prefetch_state(p)
                if not multi:
                    self.update_step(group, p, gindex, pindex)
                else:
                    u = self._update_args(group, p, gindex, pindex)
                    if u.per_parameter():
                        if self.capturable:
                            raise ValueError(_NO_TRUST_RATIO)
                        self._launch(u)
                    else:
                        updates.append(u)
                last = p
        for batch in group_updates(updates):
            self._launch_multi(batch)
        if self.is_paged and last is not None:
            torch.cuda.synchronize(last.device)  # managed memory: the host may read the state right after step()
        return loss

    def _steps_in_groups(self) -> bool:
        """A subclass that replaces update_step outside this package keeps one update_step call per parameter."""
        return type(self).update_step.__module__.split(".")[0] == __name__.split(".")[0]

    def get_config(self, gindex, pindex, group):
        config = {"betas": group["betas"], "eps": group["eps"], "weight_decay": group["weight_decay"], "lr": group["lr"],
                  "alpha": group.get("alpha", 0.0), "t_alpha": group.get("t_alpha"), "t_beta3": group.get("t_beta3"),
                  "optim_bits": self.args.optim_bits, "min_8bit_size": self.args.min_8bit_size,
                  "max_unorm": self.args.max_unorm, "skip_zeros": self.args.skip_zeros}
        if (gindex, pindex) in self.mng.index2config:
            config.update(self.mng.index2config[(gindex, pindex)])
        p = self.param_groups[gindex]["params"][pindex]
        if id(p) in self.mng.pid2config:  # override_config called after register_parameters
            config.update(self.mng.pid2config[id(p)])
        return config

    def init_state(self, group, p, gindex, pindex):
        raise NotImplementedError("init_state method needs to be overridden")

    @torch.no_grad()
    def update_step(self, group, p, gindex, pindex):
        """Update one parameter: compute its launch arguments (advancing its step) and launch them."""
        u = self._update_args(group, p, gindex, pindex)
        if not self.capturable:
            self._launch(u)
        elif u.per_parameter():
            raise ValueError(_NO_TRUST_RATIO)
        else:
            self._launch_multi([u])  # (the call advances the device step)

    def _update_args(self, group, p, gindex, pindex) -> _Update:
        raise NotImplementedError("The update_step method needs to be overridden")

    def _make_update(self, group, p, gindex, pindex):
        """Common part of _update_args: contiguous parameter and gradient, the config, the step advanced."""
        if not p.is_contiguous():
            p.data = p.data.contiguous()
        if not p.grad.is_contiguous():
            p.grad = p.grad.contiguous()
        state = self.state[p]
        if not self.capturable:  # (a capturable step is advanced on the device by the update call)
            state["step"] += 1
        return state, self.get_config(gindex, pindex, group)

    def _initial_step(self, p, step=0):
        """state["step"]: an int, or for capturable=True an int32 counter on the parameter's device."""
        return torch.tensor([step], dtype=torch.int32, device=p.device) if self.capturable else step

    def _check_capturable(self):
        """Refuse at construction what needs a host value at every step of a capturable optimizer."""
        if not self.capturable:
            return
        if self.is_paged:
            raise ValueError("capturable=True does not support paged state: its prefetch and synchronisation cannot be "
                             "captured in a CUDA graph")
        if self.args.optim_bits == 32 and self.args.max_unorm > 0.0:
            raise ValueError(_NO_TRUST_RATIO)
        if any(g.get("t_alpha") or g.get("t_beta3") for g in self.param_groups):
            raise ValueError(_NO_SCHEDULES)

    def _launch(self, u: _Update):
        st = u.state
        if st["state1"].dtype == torch.float32:
            F.optimizer_update_32bit(u.name, u.p.grad, u.p, st["state1"], u.beta1, u.eps, st["step"], u.lr, st.get("state2"),
                                     u.beta2, u.beta3, u.alpha, u.weight_decay, 1.0,
                                     st["unorm_vec"] if u.max_unorm > 0.0 else None, max_unorm=u.max_unorm,
                                     skip_zeros=u.skip_zeros)
        else:
            F.optimizer_update_8bit_blockwise(u.name, u.p.grad, u.p, st["state1"], st.get("state2"), u.beta1, u.beta2,
                                              u.beta3, u.alpha, u.eps, st["step"], u.lr, st["qmap1"], st.get("qmap2"),
                                              st["absmax1"], st.get("absmax2"), u.weight_decay, gnorm_scale=1.0,
                                              skip_zeros=u.skip_zeros)

    def _launch_multi(self, batch):
        """One multi-tensor call for updates with equal group keys."""
        u, st = batch[0], batch[0].state
        g = [b.p.grad for b in batch]
        p = [b.p for b in batch]
        s1 = [b.state["state1"] for b in batch]
        s2 = [b.state["state2"] for b in batch] if "state2" in st else None
        steps = [b.state["step"] for b in batch]
        if st["state1"].dtype == torch.float32:
            F.optimizer_update_32bit_multi(u.name, g, p, s1, u.beta1, u.eps, steps, u.lr, s2, u.beta2, u.beta3, u.alpha,
                                           u.weight_decay, 1.0, skip_zeros=u.skip_zeros)
        else:
            a1 = [b.state["absmax1"] for b in batch]
            a2 = [b.state["absmax2"] for b in batch] if s2 is not None else None
            F.optimizer_update_8bit_blockwise_multi(u.name, g, p, s1, s2, u.beta1, u.beta2, u.beta3, u.alpha, u.eps, steps,
                                                    u.lr, st["qmap1"], st.get("qmap2"), a1, a2, u.weight_decay,
                                                    gnorm_scale=1.0, skip_zeros=u.skip_zeros)

    def get_state_buffer(self, p, dtype=torch.float32):
        if p.device.type != "cuda":
            raise NotImplementedError("bitsandbytes_b200 optimizers hold their state on the GPU: there is no CPU backend")
        if not self.is_paged or p.numel() < 1e5:
            return torch.zeros_like(p, dtype=dtype, device=p.device)
        buff = F.get_paged(*p.shape, dtype=dtype, device=p.device)
        F.fill(buff, 0)
        self.page_mng.paged_tensors.append(buff)
        return buff

    def prefetch_state(self, p):
        if not self.is_paged:
            return
        state = self.state[p]
        if getattr(state["state1"], "is_paged", False):
            F.prefetch_tensor(state["state1"])
            if "state2" in state:
                F.prefetch_tensor(state["state2"])

    # ---- shared by the one- and two-state classes
    def _state_dtype(self, config, p):
        if config["optim_bits"] == 32:
            dtype = torch.float32
        elif config["optim_bits"] == 8:
            dtype = torch.uint8
        else:
            raise NotImplementedError(f"Amount of optimizer bits not supported: {config['optim_bits']}")
        return torch.float32 if p.numel() < config["min_8bit_size"] else dtype

    def _qmap(self, name, device):
        if name not in self.name2qmap:
            self.fill_qmap()
        self.name2qmap[name] = self.name2qmap[name].to(device)
        return self.name2qmap[name]

    @staticmethod
    def _blocks(p):
        return -(-p.numel() // _STATE_BLOCK)

    def _validate(self, lr, eps, betas, weight_decay):
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if isinstance(betas, str):  # '(beta1, beta2)' from a command line
            betas = [float(b) for b in betas.replace("(", "").replace(")", "").strip().split(",")]
        for i, b in enumerate(betas):
            if not 0.0 <= b < 1.0:
                raise ValueError(f"Invalid beta parameter at index {i}: {b}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        return betas

    def _set_args(self, args, optim_bits, min_8bit_size, max_unorm, skip_zeros):
        if args is None:
            args = MockArgs({"optim_bits": optim_bits, "min_8bit_size": min_8bit_size, "max_unorm": max_unorm,
                             "skip_zeros": skip_zeros})
        self.args = args


class Optimizer2State(Optimizer8bit):
    """Two moving averages per parameter: Adam / AdamW / LAMB / AdEMAMix."""

    def __init__(self, optimizer_name, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, optim_bits=32,
                 args=None, min_8bit_size=4096, max_unorm=0.0, skip_zeros=False, is_paged=False, alpha=0.0,
                 t_alpha: Optional[int] = None, t_beta3: Optional[int] = None, capturable=False):
        betas = self._validate(lr, eps, betas, weight_decay)
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, alpha=alpha, t_alpha=t_alpha,
                        t_beta3=t_beta3)
        super().__init__(params, defaults, optim_bits, is_paged, capturable)
        self._set_args(args, optim_bits, min_8bit_size, max_unorm, skip_zeros)
        self.optimizer_name = optimizer_name
        self._check_capturable()

    @torch.no_grad()
    def init_state(self, group, p, gindex, pindex):
        config = self.get_config(gindex, pindex, group)
        dtype = self._state_dtype(config, p)
        state = self.state[p]
        state["step"] = self._initial_step(p)
        state["state1"] = self.get_state_buffer(p, dtype=dtype)
        state["state2"] = self.get_state_buffer(p, dtype=dtype)
        if dtype == torch.uint8:
            state["qmap1"] = self._qmap("dynamic", p.device)
            state["qmap2"] = self._qmap("udynamic", p.device)
            state["absmax1"] = torch.zeros((self._blocks(p),), dtype=torch.float32, device=p.device)
            state["absmax2"] = torch.zeros((self._blocks(p),), dtype=torch.float32, device=p.device)
        if config["max_unorm"] > 0.0:
            state["unorm_vec"] = torch.zeros((1,), device=p.device)

    def _update_args(self, group, p, gindex, pindex) -> _Update:
        state, config = self._make_update(group, p, gindex, pindex)
        betas = config["betas"]
        beta3 = betas[2] if len(betas) >= 3 else 0.0
        return _Update(self.optimizer_name, p, state, config, betas[0], betas[1], beta3, config.get("alpha", 0.0))


class Optimizer1State(Optimizer8bit):
    """One moving average per parameter: SGD with momentum / LARS / RMSprop / Adagrad / Lion."""

    def __init__(self, optimizer_name, params, lr=1e-3, betas=(0.9, 0.0), eps=1e-8, weight_decay=0.0, optim_bits=32,
                 args=None, min_8bit_size=4096, max_unorm=0.0, skip_zeros=False, is_paged=False, capturable=False):
        betas = self._validate(lr, eps, betas, weight_decay)
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults, optim_bits, is_paged, capturable)
        self._set_args(args, optim_bits, min_8bit_size, max_unorm, skip_zeros)
        self.optimizer_name = optimizer_name
        self._check_capturable()

    @torch.no_grad()
    def init_state(self, group, p, gindex, pindex):
        config = self.get_config(gindex, pindex, group)
        dtype = self._state_dtype(config, p)
        state = self.state[p]
        state["step"] = self._initial_step(p)
        state["state1"] = self.get_state_buffer(p, dtype=dtype)
        if dtype == torch.uint8:
            state["qmap1"] = self._qmap("dynamic", p.device)
            state["absmax1"] = torch.zeros((self._blocks(p),), dtype=torch.float32, device=p.device)
        if config["max_unorm"] > 0.0:
            state["unorm_vec"] = torch.zeros((1,), device=p.device)

    def _update_args(self, group, p, gindex, pindex) -> _Update:
        state, config = self._make_update(group, p, gindex, pindex)
        return _Update(self.optimizer_name, p, state, config, config["betas"][0], config["betas"][1], 0.0, 0.0)
