"""AdEMAMix: Adam with a second, slow gradient EMA mixed into the numerator (reference
bitsandbytes/optim/ademamix.py).  Both EMAs live in ``state1`` ([2, *shape]; the 8-bit absmax is [2, blocks]);
``t_alpha`` / ``t_beta3`` are the warm-up horizons of the mixing weight and of the slow EMA's decay."""
import math
from typing import Optional

import torch

from .. import functional as F
from .optimizer import _NO_SCHEDULES, Optimizer2State, _Update


def _schedules(step, beta1, beta3, alpha, t_alpha, t_beta3):
    """Warm-up of the mixing weight (linear in the step) and of the slow EMA's decay (interpolated in log space)."""
    alpha_t = min(step * alpha / t_alpha, alpha) if t_alpha else alpha
    beta3_t = beta3
    if t_beta3:
        ln1, ln3 = math.log(beta1), math.log(beta3)
        frac = step / t_beta3
        beta3_t = min(math.exp((ln1 * ln3) / (((1 - frac) * ln3) + (frac * ln1))), beta3)
    return alpha_t, beta3_t


class _ReferenceAdEMAMix(torch.optim.Optimizer):
    """Eager PyTorch AdEMAMix with the same update order as the native kernels (csrc/optim.cu): the baseline the tests
    compare the fused optimizers with (the reference package exposes one under this name, ademamix.py:14-112)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, eps=1e-8, weight_decay=1e-2,
                 t_beta3: Optional[int] = None, t_alpha: Optional[int] = None):
        super().__init__(params, dict(lr=lr, betas=betas, alpha=alpha, eps=eps, weight_decay=weight_decay, t_beta3=t_beta3,
                                      t_alpha=t_alpha))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
            beta1, beta2, beta3 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                state = self.state[p]
                if not state:
                    state["step"] = 0
                    state["m1_m2"] = p.new_zeros((2, *p.shape))
                    state["nu"] = torch.zeros_like(p)
                state["step"] += 1
                step = state["step"]
                alpha_t, beta3_t = _schedules(step, beta1, beta3, group["alpha"], group["t_alpha"], group["t_beta3"])
                m1, m2, nu, g = state["m1_m2"][0], state["m1_m2"][1], state["nu"], p.grad
                m1.mul_(beta1).add_(g, alpha=1 - beta1)
                m2.mul_(beta3_t).add_(g, alpha=1 - beta3_t)
                nu.mul_(beta2).addcmul_(g, g, value=1 - beta2)
                c1 = 1 - beta1**step
                c2 = math.sqrt(1 - beta2**step)
                p.add_((m1 / c1 + alpha_t * m2) / (nu.sqrt() / c2 + eps), alpha=-lr)
                if wd > 0:
                    p.mul_(1 - lr * wd)
        return loss


class AdEMAMix(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha: Optional[int] = None,
                 t_beta3: Optional[int] = None, eps=1e-8, weight_decay=1e-2, optim_bits=32, min_8bit_size=4096,
                 is_paged=False, capturable=False):
        super().__init__("ademamix", params=params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                         optim_bits=optim_bits, args=None, min_8bit_size=min_8bit_size, is_paged=is_paged, alpha=alpha,
                         t_alpha=t_alpha, t_beta3=t_beta3, capturable=capturable)

    @torch.no_grad()
    def init_state(self, group, p, gindex, pindex):
        config = self.get_config(gindex, pindex, group)
        dtype = self._state_dtype(config, p)
        state = self.state[p]
        state["step"] = self._initial_step(p)
        if dtype == torch.uint8:
            state["qmap1"] = self._qmap("dynamic", p.device)
            state["qmap2"] = self._qmap("udynamic", p.device)
            state["absmax1"] = torch.zeros((2, self._blocks(p)), dtype=torch.float32, device=p.device)
            state["absmax2"] = torch.zeros((self._blocks(p),), dtype=torch.float32, device=p.device)
        state["state1"] = self._get_state_double_buffer(p, dtype=dtype)
        state["state2"] = self.get_state_buffer(p, dtype=dtype)

    def _update_args(self, group, p, gindex, pindex) -> _Update:
        u = super()._update_args(group, p, gindex, pindex)
        config = self.get_config(gindex, pindex, group)
        if config["t_alpha"] or config["t_beta3"]:  # the warm-up schedules: scalars of this parameter's step
            if self.capturable:  # (a per-parameter override: the constructor refuses the group-wide schedules)
                raise ValueError(_NO_SCHEDULES)
            u.alpha, u.beta3 = _schedules(u.state["step"], u.beta1, u.beta3, config["alpha"], config["t_alpha"],
                                          config["t_beta3"])
        return u

    def _get_state_double_buffer(self, p, dtype=torch.float32):
        if not self.is_paged or p.numel() < 1e5:
            return torch.zeros((2, *p.size()), dtype=dtype, device=p.device)
        buff = F.get_paged(*(2, *p.size()), dtype=dtype, device=p.device)
        F.fill(buff, 0)
        self.page_mng.paged_tensors.append(buff)
        return buff


class AdEMAMix8bit(AdEMAMix):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha: Optional[int] = None,
                 t_beta3: Optional[int] = None, eps=1e-8, weight_decay=1e-2, min_8bit_size=4096, is_paged=False,
                 capturable=False):
        super().__init__(params, lr=lr, betas=betas, alpha=alpha, t_alpha=t_alpha, t_beta3=t_beta3, eps=eps,
                         weight_decay=weight_decay, optim_bits=8, min_8bit_size=min_8bit_size, is_paged=is_paged,
                         capturable=capturable)


class PagedAdEMAMix8bit(AdEMAMix8bit):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha: Optional[int] = None,
                 t_beta3: Optional[int] = None, eps=1e-8, weight_decay=1e-2, min_8bit_size=4096, capturable=False):
        super().__init__(params, lr=lr, betas=betas, alpha=alpha, t_alpha=t_alpha, t_beta3=t_beta3, eps=eps,
                         weight_decay=weight_decay, min_8bit_size=min_8bit_size, is_paged=True, capturable=capturable)


class PagedAdEMAMix(AdEMAMix):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha: Optional[int] = None,
                 t_beta3: Optional[int] = None, eps=1e-8, weight_decay=1e-2, optim_bits=32, min_8bit_size=4096,
                 capturable=False):
        super().__init__(params, lr=lr, betas=betas, alpha=alpha, t_alpha=t_alpha, t_beta3=t_beta3, eps=eps,
                         weight_decay=weight_decay, optim_bits=optim_bits, min_8bit_size=min_8bit_size, is_paged=True,
                         capturable=capturable)


class AdEMAMix32bit(AdEMAMix):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha: Optional[int] = None,
                 t_beta3: Optional[int] = None, eps=1e-8, weight_decay=1e-2, min_8bit_size=4096, is_paged=False,
                 capturable=False):
        super().__init__(params, lr=lr, betas=betas, alpha=alpha, t_alpha=t_alpha, t_beta3=t_beta3, eps=eps,
                         weight_decay=weight_decay, optim_bits=32, min_8bit_size=min_8bit_size, is_paged=is_paged,
                         capturable=capturable)


class PagedAdEMAMix32bit(AdEMAMix32bit):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha: Optional[int] = None,
                 t_beta3: Optional[int] = None, eps=1e-8, weight_decay=1e-2, min_8bit_size=4096, capturable=False):
        super().__init__(params, lr=lr, betas=betas, alpha=alpha, t_alpha=t_alpha, t_beta3=t_beta3, eps=eps,
                         weight_decay=weight_decay, min_8bit_size=min_8bit_size, is_paged=True, capturable=capturable)
