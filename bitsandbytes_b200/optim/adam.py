"""Adam with 32-bit or blockwise 8-bit state (reference bitsandbytes/optim/adam.py: same constructor arguments).
``amsgrad`` exists for signature compatibility only."""
from .optimizer import Optimizer2State


def _no_amsgrad(amsgrad, who):
    if amsgrad:  # (the non-8-bit classes accept and ignore the flag, as the reference does)
        raise ValueError(f"{who} does not support amsgrad=True")


class Adam(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, is_paged=False, capturable=False):
        super().__init__("adam", params, lr, betas, eps, weight_decay, optim_bits, args, min_8bit_size,
                         is_paged=is_paged, capturable=capturable)


class Adam8bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, is_paged=False, capturable=False):
        _no_amsgrad(amsgrad, "Adam8bit")
        if optim_bits != 32:  # the argument exists for signature compatibility only (reference adam.py:120-124)
            raise ValueError("Adam8bit only supports optim_bits=32 (default value for compatibility)")
        super().__init__("adam", params, lr, betas, eps, weight_decay, 8, args, min_8bit_size, is_paged=is_paged,
                         capturable=capturable)


class Adam32bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, is_paged=False, capturable=False):
        super().__init__("adam", params, lr, betas, eps, weight_decay, 32, args, min_8bit_size, is_paged=is_paged,
                         capturable=capturable)


class PagedAdam(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, is_paged=False, capturable=False):
        super().__init__("adam", params, lr, betas, eps, weight_decay, optim_bits, args, min_8bit_size, is_paged=True,
                         capturable=capturable)


class PagedAdam8bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, is_paged=False, capturable=False):
        _no_amsgrad(amsgrad, "PagedAdam8bit")
        if optim_bits != 32:
            raise ValueError("PagedAdam8bit only supports optim_bits=32 (default value for compatibility)")
        super().__init__("adam", params, lr, betas, eps, weight_decay, 8, args, min_8bit_size, is_paged=True,
                         capturable=capturable)


class PagedAdam32bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, is_paged=False, capturable=False):
        super().__init__("adam", params, lr, betas, eps, weight_decay, 32, args, min_8bit_size, is_paged=True,
                         capturable=capturable)
