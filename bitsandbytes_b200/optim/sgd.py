"""SGD with momentum (reference bitsandbytes/optim/sgd.py; plain SGD keeps no state and is not provided there either)."""
from .optimizer import Optimizer1State


def _need_momentum(momentum):
    if momentum == 0:
        raise NotImplementedError("SGD without momentum is not supported!")


class SGD(Optimizer1State):
    def __init__(self, params, lr, momentum=0, dampening=0, weight_decay=0, nesterov=False, optim_bits=32, args=None,
                 min_8bit_size=4096, capturable=False):
        _need_momentum(momentum)
        super().__init__("momentum", params, lr, (momentum, dampening), 0.0, weight_decay, optim_bits, args,
                         min_8bit_size, capturable=capturable)


class SGD8bit(Optimizer1State):
    def __init__(self, params, lr, momentum=0, dampening=0, weight_decay=0, nesterov=False, args=None,
                 min_8bit_size=4096, capturable=False):
        _need_momentum(momentum)
        super().__init__("momentum", params, lr, (momentum, dampening), 0.0, weight_decay, 8, args, min_8bit_size,
                         capturable=capturable)


class SGD32bit(Optimizer1State):
    def __init__(self, params, lr, momentum=0, dampening=0, weight_decay=0, nesterov=False, args=None,
                 min_8bit_size=4096, capturable=False):
        _need_momentum(momentum)
        super().__init__("momentum", params, lr, (momentum, dampening), 0.0, weight_decay, 32, args, min_8bit_size,
                         capturable=capturable)
