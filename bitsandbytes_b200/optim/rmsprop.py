"""RMSprop (reference bitsandbytes/optim/rmsprop.py)."""
from .optimizer import Optimizer1State


def _check(alpha, centered):
    if alpha == 0:
        raise NotImplementedError("RMSprop with alpha==0.0 is not supported!")
    if centered:
        raise NotImplementedError("Centered RMSprop is not supported!")


class RMSprop(Optimizer1State):
    def __init__(self, params, lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0, momentum=0, centered=False, optim_bits=32,
                 args=None, min_8bit_size=4096, capturable=False):
        _check(alpha, centered)
        super().__init__("rmsprop", params, lr, (alpha, momentum), eps, weight_decay, optim_bits, args, min_8bit_size,
                         capturable=capturable)


class RMSprop8bit(Optimizer1State):
    def __init__(self, params, lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0, momentum=0, centered=False, args=None,
                 min_8bit_size=4096, capturable=False):
        _check(alpha, centered)
        super().__init__("rmsprop", params, lr, (alpha, momentum), eps, weight_decay, 8, args, min_8bit_size,
                         capturable=capturable)


class RMSprop32bit(Optimizer1State):
    def __init__(self, params, lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0, momentum=0, centered=False, args=None,
                 min_8bit_size=4096, capturable=False):
        _check(alpha, centered)
        super().__init__("rmsprop", params, lr, (alpha, momentum), eps, weight_decay, 32, args, min_8bit_size,
                         capturable=capturable)
