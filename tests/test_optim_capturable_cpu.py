"""CPU checks of the capturable optimizer step's host logic: the descriptor union, what the capturable native calls are
given (step-counter and lr pointers, capacity chunks), the capturable= keyword of every optimizer class, what a
capturable optimizer refuses, and the capture guard of step()."""
import ctypes as ct

import pytest
import torch

import bitsandbytes_b200 as bnb
from bitsandbytes_b200 import cextension as cext
from bitsandbytes_b200.backends import cuda as backend
from bitsandbytes_b200.optim.optimizer import _Update, group_updates


def test_the_step_pointer_shares_the_last_8_bytes_of_the_64_byte_descriptor():
    assert ct.sizeof(cext.OptimTensor) == 64
    assert cext.OptimTensor.step.offset == 56 and cext.OptimTensor.reserved.offset == 60
    d = cext.OptimTensor(n=5, step=3)
    assert d.step_ptr == 3  # (little endian: step is the low half, reserved the high half)
    d.step_ptr = 0x7F12_3456_7890
    assert (d.step, d.reserved) == (0x3456_7890, 0x7F12) and d.step_ptr == 0x7F12_3456_7890 and d.n == 5
    # the capacity of a launch is that of the integer-step entries: the 448-tensor LoRA set of a Llama-3-8B still fits
    assert backend.optimizer_multi_capacity() == 453
    for name in ("cbnb_b200_optimizer_update_32bit_multi_dev", "cbnb_b200_optimizer_update_8bit_blockwise_multi_dev"):
        assert name in cext.EXPORTED_SYMBOLS


class _OnCuda(torch.Tensor):
    """A CPU tensor that reports cuda:0: exercises the host packing of the capturable route without a GPU."""

    @property
    def device(self):
        return torch.device("cuda", 0)

    @property
    def is_cuda(self):
        return True


def _cuda(t):
    return torch.Tensor._make_subclass(_OnCuda, t)


class _FakeLib:
    """Records the native multi calls instead of launching: per call, the descriptors' (n, step, step_ptr) and the
    arguments after the descriptor count."""

    def __init__(self, cap):
        self.cap, self.calls = cap, []

    def cbnb_b200_optimizer_multi_capacity(self):
        return self.cap

    def _record(self, name):
        def call(opt, dtype, tensors, count, *rest):
            descs = (cext.OptimTensor * count).from_address(tensors)
            self.calls.append((name, [(d.n, d.step, d.step_ptr) for d in descs], rest))
            return 0
        return call

    def __getattr__(self, name):
        if name.startswith("cbnb_b200_optimizer_update"):
            return self._record(name)
        raise AttributeError(name)

    def check(self, what):
        pass


@pytest.fixture
def fake(monkeypatch):
    lib = _FakeLib(cap=7)
    monkeypatch.setattr(backend, "lib", lib)
    monkeypatch.setattr(backend, "_multi_capacity", None)
    monkeypatch.setattr(backend, "_stream", lambda t: 0)
    return lib


def _lists(k, bits):
    g = [_cuda(torch.zeros(i + 1, dtype=torch.bfloat16)) for i in range(k)]
    p = [_cuda(torch.zeros(i + 1, dtype=torch.bfloat16)) for i in range(k)]
    s1 = [_cuda(torch.zeros(i + 1, dtype=torch.uint8 if bits == 8 else torch.float32)) for i in range(k)]
    a1 = [_cuda(torch.zeros(1)) for _ in range(k)]
    steps = [_cuda(torch.zeros(1, dtype=torch.int32)) for _ in range(k)]
    return g, p, s1, a1, steps


def _call(bits, g, p, s1, a1, steps, lr):
    if bits == 8:
        backend.optimizer_update_8bit_blockwise_multi("lion", g, p, s1, None, 0.9, 0.99, 0.0, 0.0, 0.0, steps, lr,
                                                      _cuda(torch.zeros(256)), None, a1, None, 0.0)
    else:
        backend.optimizer_update_32bit_multi("lion", g, p, s1, None, 0.9, 0.99, 0.0, 0.0, 0.0, 0.0, steps, lr)


@pytest.mark.parametrize("bits", [8, 32])
@pytest.mark.parametrize("k", [1, 7, 8, 22])
def test_the_capturable_call_packs_the_step_counters_and_chunks_as_before(fake, bits, k):
    g, p, s1, a1, steps = _lists(k, bits)
    lr = _cuda(torch.tensor(3e-4))
    _call(bits, g, p, s1, a1, steps, lr)
    want = ("cbnb_b200_optimizer_update_8bit_blockwise_multi_dev" if bits == 8
            else "cbnb_b200_optimizer_update_32bit_multi_dev")
    assert [name for name, _, _ in fake.calls] == [want] * len(fake.calls)
    assert [len(d) for _, d, _ in fake.calls] == [7] * (k // 7) + ([k % 7] if k % 7 else [])
    packed = [d for _, ds, _ in fake.calls for d in ds]
    assert [n for n, _, _ in packed] == list(range(1, k + 1)), "every descriptor once, in order"
    assert [ptr for _, _, ptr in packed] == [s.data_ptr() for s in steps]
    for _, _, rest in fake.calls:  # (beta1, beta2, beta3, alpha, eps, weight_decay, lr, lr_dev, ...)
        assert rest[6] == 0.0 and rest[7] == lr.data_ptr()


@pytest.mark.parametrize("bits", [8, 32])
def test_a_float_lr_with_device_steps_is_passed_by_value(fake, bits):
    g, p, s1, a1, steps = _lists(3, bits)
    _call(bits, g, p, s1, a1, steps, 2e-3)
    (_, _, rest), = fake.calls
    assert rest[6] == pytest.approx(2e-3) and rest[7] is None


@pytest.mark.parametrize("bits", [8, 32])
def test_integer_steps_keep_the_integer_entry(fake, bits):
    g, p, s1, a1, _ = _lists(3, bits)
    _call(bits, g, p, s1, a1, [4, 5, 6], 2e-3)
    (name, descs, rest), = fake.calls
    assert not name.endswith("_dev") and [s for _, s, _ in descs] == [4, 5, 6]
    assert rest[6] == pytest.approx(2e-3) and len(rest) == (12 if bits == 8 else 10)  # (the scalars and the stream)


@pytest.mark.parametrize("bad", ["int64", "two_elements", "cpu", "shared", "mixed"])
def test_the_capturable_call_refuses_malformed_step_counters(fake, bad):
    g, p, s1, a1, steps = _lists(3, 32)
    if bad == "int64":
        steps[1] = _cuda(torch.zeros(1, dtype=torch.int64))
    elif bad == "two_elements":
        steps[1] = _cuda(torch.zeros(2, dtype=torch.int32))
    elif bad == "cpu":
        steps[1] = torch.zeros(1, dtype=torch.int32)
    elif bad == "shared":
        steps[2] = steps[0]
    else:
        steps[1] = 7
    with pytest.raises(ValueError, match="step"):
        _call(32, g, p, s1, a1, steps, 1e-3)
    assert fake.calls == []


@pytest.mark.parametrize("bad", ["float64", "two_elements", "cpu"])
def test_the_capturable_call_refuses_an_lr_tensor_that_is_not_one_fp32_on_the_device(fake, bad):
    g, p, s1, a1, steps = _lists(2, 8)
    lr = {"float64": _cuda(torch.tensor(1e-3, dtype=torch.float64)), "two_elements": _cuda(torch.tensor([1e-3, 1e-3])),
          "cpu": torch.tensor(1e-3)}[bad]
    with pytest.raises(ValueError, match="lr"):
        _call(8, g, p, s1, a1, steps, lr)
    assert fake.calls == []


# ------------------------------------------------------------------------------------------ the optimizer classes
PUBLIC = ["Adam", "Adam8bit", "Adam32bit", "AdamW", "AdamW8bit", "AdamW32bit", "Lion", "Lion8bit", "Lion32bit", "SGD",
          "SGD8bit", "SGD32bit", "RMSprop", "RMSprop8bit", "RMSprop32bit", "Adagrad", "Adagrad8bit", "Adagrad32bit",
          "AdEMAMix", "AdEMAMix8bit", "AdEMAMix32bit", "LAMB8bit", "LARS8bit"]
PAGED = ["PagedAdam", "PagedAdam8bit", "PagedAdam32bit", "PagedAdamW", "PagedAdamW8bit", "PagedAdamW32bit", "PagedLion",
         "PagedLion8bit", "PagedLion32bit", "PagedAdEMAMix", "PagedAdEMAMix8bit", "PagedAdEMAMix32bit"]
TRUST_RATIO = ["LAMB", "LAMB32bit", "LARS", "LARS32bit"]


def _kw(name):
    return dict(lr=0.1, momentum=0.9) if name.startswith(("SGD", "LARS")) else {}


def _param():
    return [torch.nn.Parameter(torch.zeros(8))]


@pytest.mark.parametrize("name", PUBLIC)
def test_every_public_class_takes_capturable(name):
    cls = getattr(bnb.optim, name)
    assert cls(_param(), **_kw(name), capturable=True).capturable
    assert not cls(_param(), **_kw(name)).capturable


@pytest.mark.parametrize("name", PAGED + TRUST_RATIO)
def test_paged_state_and_32bit_trust_ratios_are_refused_at_construction(name):
    cls = getattr(bnb.optim, name)
    assert not cls(_param(), **_kw(name), capturable=False).capturable
    with pytest.raises(ValueError, match="capturable=True does not support (paged state|32-bit state with max_unorm)"):
        cls(_param(), **_kw(name), capturable=True)


@pytest.mark.parametrize("schedule", [dict(t_alpha=100), dict(t_beta3=100)])
def test_ademamix_schedules_are_refused_at_construction(schedule):
    for cls in (bnb.optim.AdEMAMix, bnb.optim.AdEMAMix8bit):
        with pytest.raises(ValueError, match="t_alpha / t_beta3"):
            cls(_param(), capturable=True, **schedule)


def test_a_32bit_trust_ratio_from_a_per_parameter_override_is_refused_at_the_first_step(monkeypatch):
    """LAMB8bit keeps 32-bit state for a parameter below min_8bit_size: that parameter would need its norm on the
    host.  (State creation is replaced by a CPU stand-in.)"""
    p = torch.nn.Parameter(torch.zeros(8))
    p.grad = torch.zeros(8)
    opt = bnb.optim.LAMB8bit([p], capturable=True)
    monkeypatch.setattr(opt, "get_state_buffer", lambda p, dtype=torch.float32: torch.zeros_like(p, dtype=dtype))
    with pytest.raises(ValueError, match="max_unorm"):
        opt.step()


_DYN, _UDYN = torch.zeros(256), torch.zeros(256)


def test_a_tensor_lr_groups_by_identity():
    def update(lr):
        p = torch.zeros(300, dtype=torch.bfloat16)
        state = {"step": torch.zeros(1, dtype=torch.int32), "state1": torch.zeros(300, dtype=torch.uint8),
                 "qmap1": _DYN, "qmap2": _UDYN}
        return _Update("adam", p, state, dict(eps=1e-8, weight_decay=0.0, lr=lr, skip_zeros=False, max_unorm=0.0),
                       0.9, 0.999, 0.0, 0.0)

    lr_a, lr_b = torch.tensor(1e-3), torch.tensor(1e-3)
    a, b, c, d = update(lr_a), update(lr_b), update(lr_a), update(1e-3)
    assert group_updates([a, b, c, d]) == [[a, c], [b], [d]]



@pytest.fixture
def capturing(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)


def test_capturing_the_step_of_a_non_capturable_optimizer_raises(capturing):
    p = torch.nn.Parameter(torch.zeros(8))
    p.grad = torch.zeros(8)
    with pytest.raises(RuntimeError, match="capturable=False"):
        bnb.optim.AdamW8bit([p]).step()


def test_capturing_a_step_that_would_create_state_raises(capturing):
    p = torch.nn.Parameter(torch.zeros(8))
    p.grad = torch.zeros(8)
    opt = bnb.optim.AdamW8bit([p], capturable=True)
    with pytest.raises(RuntimeError, match="run one eager step"):
        opt.step()
    assert len(opt.state[p]) == 0
