"""LARS: SGD with momentum whose update norm is clipped to max_unorm x the parameter norm (reference
bitsandbytes/optim/lars.py), plus the pure-PyTorch LARS the reference ships for comparison."""
import torch
from torch.optim import Optimizer

from .optimizer import Optimizer1State


def _need_momentum(momentum):
    if momentum == 0:
        raise NotImplementedError("LARS without momentum is not supported!")


class LARS(Optimizer1State):
    def __init__(self, params, lr, momentum=0, dampening=0, weight_decay=0, nesterov=False, optim_bits=32, args=None,
                 min_8bit_size=4096, max_unorm=0.02, capturable=False):
        _need_momentum(momentum)
        super().__init__("lars", params, lr, (momentum, dampening), 0.0, weight_decay, optim_bits, args, min_8bit_size,
                         max_unorm=max_unorm, capturable=capturable)


class LARS8bit(Optimizer1State):
    def __init__(self, params, lr, momentum=0, dampening=0, weight_decay=0, nesterov=False, args=None, min_8bit_size=4096,
                 max_unorm=0.02, capturable=False):
        _need_momentum(momentum)
        super().__init__("lars", params, lr, (momentum, dampening), 0.0, weight_decay, 8, args, min_8bit_size,
                         max_unorm=max_unorm, capturable=capturable)


class LARS32bit(Optimizer1State):
    def __init__(self, params, lr, momentum=0, dampening=0, weight_decay=0, nesterov=False, args=None, min_8bit_size=4096,
                 max_unorm=0.02, capturable=False):
        _need_momentum(momentum)
        super().__init__("lars", params, lr, (momentum, dampening), 0.0, weight_decay, 32, args, min_8bit_size,
                         max_unorm=max_unorm, capturable=capturable)


class PytorchLARS(Optimizer):
    """Eager PyTorch LARS (no native kernel): momentum SGD with a per-tensor trust ratio."""

    def __init__(self, params, lr=0.01, momentum=0, dampening=0, weight_decay=0, nesterov=False, max_unorm=0.02):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay,
                                      nesterov=nesterov, max_unorm=max_unorm))

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("nesterov", False)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                d_p = p.grad
                if group["weight_decay"] != 0:
                    d_p = d_p.add(p, alpha=group["weight_decay"])
                update = d_p
                if group["momentum"] != 0:
                    buf = self.state[p].get("momentum_buffer")
                    if buf is None:
                        buf = self.state[p]["momentum_buffer"] = torch.clone(d_p).detach()
                    else:
                        buf.mul_(group["momentum"]).add_(d_p, alpha=1 - group["dampening"])
                    update = d_p + buf * group["momentum"] if group["nesterov"] else buf
                scale = 1.0
                if group["max_unorm"] > 0.0:
                    pnorm = torch.norm(p.detach())
                    unorm = torch.norm(update)
                    if unorm > group["max_unorm"] * pnorm:
                        scale = group["max_unorm"] * pnorm / unorm
                p.add_(update, alpha=-group["lr"] * scale)
        return loss
