"""CPU checks of the multi-tensor optimizer step's host logic: which parameters share a launch (group keys), which keep
one launch each, and how the backend splits a group into launches of at most the descriptor capacity."""
import ctypes as ct

import pytest
import torch

import bitsandbytes_b200 as bnb
from bitsandbytes_b200 import cextension as cext
from bitsandbytes_b200.backends import cuda as backend
from bitsandbytes_b200.optim.optimizer import _Update, group_updates

CONFIG = dict(eps=1e-8, weight_decay=0.01, lr=1e-3, skip_zeros=False, max_unorm=0.0)
DYN, UDYN = torch.zeros(256), torch.zeros(256)


def _update(n=300, dtype=torch.bfloat16, bits=8, name="adam", qmap1=DYN, qmap2=UDYN, beta3=0.0, alpha=0.0, **config):
    p = torch.zeros(n, dtype=dtype)
    state = {"step": 1, "state1": torch.zeros(n, dtype=torch.uint8 if bits == 8 else torch.float32)}
    if bits == 8:
        state.update(qmap1=qmap1, qmap2=qmap2)
    return _Update(name, p, state, dict(CONFIG, **config), 0.9, 0.999, beta3, alpha)


def test_equal_launch_arguments_share_a_group_in_order_of_first_appearance():
    a, b, c = _update(10), _update(5000), _update(7)
    other_lr = _update(10, lr=2e-3)
    d = _update(11)
    groups = group_updates([a, other_lr, b, c, d])
    assert groups == [[a, b, c, d], [other_lr]]


@pytest.mark.parametrize("field", ["dtype", "bits", "name", "lr", "weight_decay", "eps", "skip_zeros", "beta3", "alpha",
                                   "qmap"])
def test_every_per_launch_argument_is_part_of_the_group_key(field):
    changed = {"dtype": dict(dtype=torch.float32), "bits": dict(bits=32), "name": dict(name="ademamix"),
               "lr": dict(lr=5e-4), "weight_decay": dict(weight_decay=0.0), "eps": dict(eps=1e-6),
               "skip_zeros": dict(skip_zeros=True), "beta3": dict(beta3=0.9999), "alpha": dict(alpha=5.0),
               "qmap": dict(qmap1=DYN.clone())}[field]
    assert len(group_updates([_update(), _update(**changed)])) == 2


def test_the_step_of_a_parameter_does_not_split_a_group():
    a, b = _update(), _update()
    b.state["step"] = 17
    assert len(group_updates([a, b])) == 1


def test_only_32bit_state_with_a_trust_ratio_takes_the_per_parameter_route():
    assert _update(bits=32, max_unorm=1.0).per_parameter()  # LAMB / LARS: a norm pre-pass and torch.norm(p)
    assert not _update(bits=32).per_parameter()
    assert not _update(bits=8, max_unorm=1.0).per_parameter()  # (the 8-bit update has no trust ratio)


def test_a_subclass_that_replaces_update_step_keeps_the_per_parameter_loop():
    p = [torch.nn.Parameter(torch.zeros(8))]

    class Custom(bnb.optim.AdamW8bit):
        def update_step(self, group, p, gindex, pindex):
            super().update_step(group, p, gindex, pindex)

    class OnlyInit(bnb.optim.AdamW8bit):
        def init_state(self, group, p, gindex, pindex):
            super().init_state(group, p, gindex, pindex)

    assert not Custom(p)._steps_in_groups()
    assert OnlyInit(p)._steps_in_groups()
    for cls in (bnb.optim.AdamW8bit, bnb.optim.PagedAdamW8bit, bnb.optim.AdEMAMix8bit, bnb.optim.Lion, bnb.optim.LAMB,
                bnb.optim.SGD8bit, bnb.optim.RMSprop, bnb.optim.Adagrad8bit):
        kw = dict(lr=0.1, momentum=0.9) if cls is bnb.optim.SGD8bit else {}
        assert cls(p, **kw)._steps_in_groups(), cls


def test_the_descriptor_matches_the_c_header_and_a_launch_fits_the_kernel_parameter_space():
    assert ct.sizeof(cext.OptimTensor) == 64
    assert [f for f, _ in cext.OptimTensor._fields_] == ["p", "g", "state1", "state2", "absmax1", "absmax2", "n", "step",
                                                         "reserved"]
    cap = backend.optimizer_multi_capacity()
    assert 448 <= cap and cap * (64 + 8) + 16 <= 32764  # (descriptor + 8-byte work-item prefix per tensor)
    for name in ("cbnb_b200_optimizer_multi_capacity", "cbnb_b200_optimizer_update_32bit_multi",
                 "cbnb_b200_optimizer_update_8bit_blockwise_multi"):
        assert name in cext.EXPORTED_SYMBOLS


class _FakeLib:
    """Records the native multi calls instead of launching: (count, element counts of the descriptors passed)."""

    def __init__(self, cap):
        self.cap, self.calls = cap, []

    def cbnb_b200_optimizer_multi_capacity(self):
        return self.cap

    def call(self, opt, dtype, tensors, count, *rest):
        descs = (cext.OptimTensor * count).from_address(tensors)
        self.calls.append([d.n for d in descs])
        return 0

    def check(self, what):
        pass


@pytest.mark.parametrize("k", [0, 1, 6, 7, 8, 22])
def test_a_group_is_split_into_launches_of_at_most_the_capacity(monkeypatch, k):
    fake = _FakeLib(cap=7)
    monkeypatch.setattr(backend, "lib", fake)
    monkeypatch.setattr(backend, "_multi_capacity", None)
    monkeypatch.setattr(backend, "_stream", lambda t: 0)
    descs = (cext.OptimTensor * k)(*[cext.OptimTensor(n=i + 1) for i in range(k)])
    backend._launch_list("test", fake.call, "adam", torch.zeros(1, dtype=torch.bfloat16), descs, ())
    assert [len(c) for c in fake.calls] == [7] * (k // 7) + ([k % 7] if k % 7 else [])
    assert [n for c in fake.calls for n in c] == list(range(1, k + 1)), "every descriptor once, in order"


def test_mismatched_lists_and_cpu_tensors_are_refused_before_any_launch():
    g = [torch.zeros(4, dtype=torch.bfloat16)] * 2
    with pytest.raises(ValueError, match="one entry per parameter"):
        backend.optimizer_update_32bit_multi("adam", g, g, [torch.zeros(4)] * 2, [torch.zeros(4)], 0.9, 0.999, 0.0, 0.0,
                                             1e-8, 0.0, [1, 1], 1e-3)
    with pytest.raises(ValueError, match="Unsupported optimizer"):
        backend.optimizer_update_8bit_blockwise_multi("lamb", g, g, [torch.zeros(4, dtype=torch.uint8)] * 2, None, 0.9,
                                                      0.999, 0.0, 0.0, 1e-8, [1, 1], 1e-3, DYN, None,
                                                      [torch.zeros(1)] * 2, None, 0.0)
    with pytest.raises(RuntimeError, match="CUDA device"):
        backend.optimizer_update_32bit_multi("momentum", g, g, [torch.zeros(4)] * 2, None, 0.9, 0.0, 0.0, 0.0, 1e-8, 0.0,
                                             [1, 1], 1e-3)
    backend.optimizer_update_32bit_multi("momentum", [], [], [], None, 0.9, 0.0, 0.0, 0.0, 1e-8, 0.0, [], 1e-3)
