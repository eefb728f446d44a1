"""LAMB: Adam with the update norm clipped to max_unorm x the parameter norm (reference bitsandbytes/optim/lamb.py)."""
from .adam import _no_amsgrad
from .optimizer import Optimizer2State


class LAMB(Optimizer2State):
    def __init__(self, params, lr=1e-3, bias_correction=True, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False,
                 adam_w_mode=True, optim_bits=32, args=None, min_8bit_size=4096, max_unorm=1.0, capturable=False):
        super().__init__("lamb", params, lr, betas, eps, weight_decay, optim_bits, args, min_8bit_size,
                         max_unorm=max_unorm, capturable=capturable)


class LAMB8bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, bias_correction=True, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False,
                 adam_w_mode=True, args=None, min_8bit_size=4096, max_unorm=1.0, capturable=False):
        _no_amsgrad(amsgrad, "LAMB8bit")
        if max_unorm != 1.0:  # the blockwise 8-bit update has no update-norm clipping: refuse what would be ignored
            raise ValueError("LAMB8bit only supports max_unorm=1.0 (default value for compatibility)")
        super().__init__("lamb", params, lr, betas, eps, weight_decay, 8, args, min_8bit_size, max_unorm=max_unorm,
                         capturable=capturable)


class LAMB32bit(Optimizer2State):
    def __init__(self, params, lr=1e-3, bias_correction=True, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False,
                 adam_w_mode=True, args=None, min_8bit_size=4096, max_unorm=1.0, capturable=False):
        super().__init__("lamb", params, lr, betas, eps, weight_decay, 32, args, min_8bit_size, max_unorm=max_unorm,
                         capturable=capturable)
