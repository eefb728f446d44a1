"""AdamW (decoupled weight decay, default 0.01) with 32-bit or blockwise 8-bit state (reference
bitsandbytes/optim/adamw.py).  The update is the Adam kernel: its weight decay is already the decoupled form."""
from .adam import _no_amsgrad
from .optimizer import Optimizer2State


class AdamW(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, is_paged=False, capturable=False):
        super().__init__("adam", params, lr, betas, eps, weight_decay, optim_bits, args, min_8bit_size,
                         is_paged=is_paged, capturable=capturable)


class AdamW8bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, is_paged=False, capturable=False):
        _no_amsgrad(amsgrad, "AdamW8bit")
        if optim_bits != 32:
            raise ValueError("AdamW8bit only supports optim_bits=32 (default value for compatibility)")
        super().__init__("adam", params, lr, betas, eps, weight_decay, 8, args, min_8bit_size, is_paged=is_paged,
                         capturable=capturable)


class AdamW32bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, is_paged=False, capturable=False):
        super().__init__("adam", params, lr, betas, eps, weight_decay, 32, args, min_8bit_size, is_paged=is_paged,
                         capturable=capturable)


class PagedAdamW(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, capturable=False):
        super().__init__("adam", params, lr, betas, eps, weight_decay, optim_bits, args, min_8bit_size, is_paged=True,
                         capturable=capturable)


class PagedAdamW8bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, capturable=False):
        _no_amsgrad(amsgrad, "PagedAdamW8bit")
        if optim_bits != 32:
            raise ValueError("PagedAdamW8bit only supports optim_bits=32 (default value for compatibility)")
        super().__init__("adam", params, lr, betas, eps, weight_decay, 8, args, min_8bit_size, is_paged=True,
                         capturable=capturable)


class PagedAdamW32bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32,
                 args=None, min_8bit_size=4096, capturable=False):
        super().__init__("adam", params, lr, betas, eps, weight_decay, 32, args, min_8bit_size, is_paged=True,
                         capturable=capturable)
