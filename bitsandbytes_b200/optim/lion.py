"""Lion (sign of the interpolated momentum, decoupled weight decay) -- reference bitsandbytes/optim/lion.py."""
from .optimizer import Optimizer1State


class Lion(Optimizer1State):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, optim_bits=32, args=None, min_8bit_size=4096,
                 is_paged=False, capturable=False):
        super().__init__("lion", params, lr, betas, 0.0, weight_decay, optim_bits, args, min_8bit_size,
                         is_paged=is_paged, capturable=capturable)


class Lion8bit(Optimizer1State):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, args=None, min_8bit_size=4096,
                 is_paged=False, capturable=False):
        super().__init__("lion", params, lr, betas, 0.0, weight_decay, 8, args, min_8bit_size, is_paged=is_paged,
                         capturable=capturable)


class Lion32bit(Optimizer1State):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, args=None, min_8bit_size=4096,
                 is_paged=False, capturable=False):
        super().__init__("lion", params, lr, betas, 0.0, weight_decay, 32, args, min_8bit_size, is_paged=is_paged,
                         capturable=capturable)


class PagedLion(Optimizer1State):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, optim_bits=32, args=None,
                 min_8bit_size=4096, capturable=False):
        super().__init__("lion", params, lr, betas, 0.0, weight_decay, optim_bits, args, min_8bit_size, is_paged=True,
                         capturable=capturable)


class PagedLion8bit(Optimizer1State):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, args=None, min_8bit_size=4096,
                 capturable=False):
        super().__init__("lion", params, lr, betas, 0.0, weight_decay, 8, args, min_8bit_size, is_paged=True,
                         capturable=capturable)


class PagedLion32bit(Optimizer1State):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, args=None, min_8bit_size=4096,
                 capturable=False):
        super().__init__("lion", params, lr, betas, 0.0, weight_decay, 32, args, min_8bit_size, is_paged=True,
                         capturable=capturable)
