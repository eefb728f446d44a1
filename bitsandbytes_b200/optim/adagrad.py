"""Adagrad (reference bitsandbytes/optim/adagrad.py)."""
from .optimizer import Optimizer1State


def _check(lr, weight_decay, eps, initial_accumulator_value, lr_decay):
    if not 0.0 <= lr:
        raise ValueError(f"Invalid learning rate: {lr}")
    if not 0.0 <= weight_decay:
        raise ValueError(f"Invalid weight_decay value: {weight_decay}")
    if not 0.0 <= eps:
        raise ValueError(f"Invalid epsilon value: {eps}")
    if initial_accumulator_value != 0.0:
        raise ValueError("Initial accumulator value != 0.0 not supported!")
    if lr_decay != 0.0:
        raise ValueError("Lr Decay != 0.0 not supported!")


class Adagrad(Optimizer1State):
    def __init__(self, params, lr=1e-2, lr_decay=0, weight_decay=0, initial_accumulator_value=0, eps=1e-10, optim_bits=32,
                 args=None, min_8bit_size=4096, capturable=False):
        _check(lr, weight_decay, eps, initial_accumulator_value, lr_decay)
        super().__init__("adagrad", params, lr, (0.0, 0.0), eps, weight_decay, optim_bits, args, min_8bit_size,
                         capturable=capturable)


class Adagrad8bit(Optimizer1State):
    def __init__(self, params, lr=1e-2, lr_decay=0, weight_decay=0, initial_accumulator_value=0, eps=1e-10, optim_bits=8,
                 args=None, min_8bit_size=4096, capturable=False):
        _check(lr, weight_decay, eps, initial_accumulator_value, lr_decay)
        if optim_bits != 8:
            raise ValueError("Adagrad8bit only supports optim_bits=8 (default value for compatibility)")
        super().__init__("adagrad", params, lr, (0.0, 0.0), eps, weight_decay, 8, args, min_8bit_size,
                         capturable=capturable)


class Adagrad32bit(Optimizer1State):
    def __init__(self, params, lr=1e-2, lr_decay=0, weight_decay=0, initial_accumulator_value=0, eps=1e-10, optim_bits=32,
                 args=None, min_8bit_size=4096, capturable=False):
        _check(lr, weight_decay, eps, initial_accumulator_value, lr_decay)
        super().__init__("adagrad", params, lr, (0.0, 0.0), eps, weight_decay, 32, args, min_8bit_size,
                         capturable=capturable)
