"""The simulated tensor-parallel world of the CPU tests, shared by the test files that import it (a plain module: the
fixtures below become a file's own by import).

* :class:`FakeLib` stands in for the native library: it records every ``cbnb_b200_*`` call and serves it, or refuses
  the names in ``refuse`` (a non-zero return code).
* :func:`simulate` makes this process rank ``rank`` of a world of ``world``: the NCCL collectives record their shapes
  and copy (an all-gather repeats this rank's input for every rank), and symmetric memory hands out buffers whose peer
  addresses are made up (:func:`peer_ptrs`) and whose peer copies and barriers are recorded (:class:`Handle`)."""
import ctypes as ct

import pytest
import torch

import bitsandbytes_b200.backends.cuda as cb
import bitsandbytes_b200.parallel as par

# the argument index of the destination array (its length follows it) of the multi-destination native calls
_DEST_ARG = {"cbnb_b200_gemm_4bit_multi_out": 6, "cbnb_b200_gemm_4bit_partial": 6,
             "cbnb_b200_gemm_4bit_partial_scatter": 6, "cbnb_b200_int8_gemm_multi_out": 8,
             "cbnb_b200_int8_gemm_partial_scatter": 2}
_FAKE_ADDRS = 100_000_000  # peer_ptrs stay below this; a host tensor's address does not


def peer_ptrs(slot: int, world: int) -> list[int]:
    """The made-up base address of every rank's buffer of symmetric-memory slot ``slot`` (numbered as allocated)."""
    return [(slot + 1) * 1_000_000 + r * 10_000 for r in range(world)]


class FakeLib:
    """Records every native call as ``(name, args)`` in ``calls`` and the destination list of a multi-destination call,
    read while the call is made, in ``dests``.  With ``log``, each call is also appended there as ``(name without the
    prefix, its scalar arguments, its destinations)``, a destination that is a host tensor shown as ``"t"``."""

    def __init__(self, log=None):
        self.calls, self.dests, self.refuse, self.log = [], [], set(), log

    def __getattr__(self, name):
        if not name.startswith("cbnb_b200_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name, args))
            dests = None
            if name in _DEST_ARG:
                i = _DEST_ARG[name]
                arr = ct.cast(args[i], ct.POINTER(ct.c_void_p))
                self.dests.append([arr[j] for j in range(args[i + 1])])
                dests = [p if p < _FAKE_ADDRS else "t" for p in self.dests[-1]]
            if self.log is not None:
                scalars = tuple(a for a in args if isinstance(a, (int, float)) and abs(a) < _FAKE_ADDRS)
                self.log.append((name[len("cbnb_b200_"):], scalars, dests))
            return 1 if name in self.refuse else 0
        return call

    def names(self) -> list[str]:
        return [n for n, _ in self.calls]

    def check(self, what=""):
        pass


def install_fake_lib(monkeypatch, log=None) -> FakeLib:
    lib = FakeLib(log)
    monkeypatch.setattr(cb, "lib", lib)
    monkeypatch.setattr(cb, "_stream", lambda t: 0)
    return lib


@pytest.fixture
def fake(monkeypatch):
    return install_fake_lib(monkeypatch)


class Handle:
    """The symmetric-memory handle of slot ``slot``: peer copies and barriers appended to ``log`` and counted."""

    def __init__(self, world, rank, slot, log):
        self.world_size, self.rank, self.slot, self.log = world, rank, slot, log
        self.buffer_ptrs = peer_ptrs(slot, world)
        self.barriers = 0

    def get_buffer(self, r, shape, dtype, offset):
        self.log.append(("copy", self.slot, r, tuple(shape), dtype, offset))
        return torch.zeros(shape, dtype=dtype)

    def barrier(self, channel=0):
        self.barriers += 1
        self.log.append(("barrier", self.slot))


def simulate(monkeypatch, world: int, rank: int, log: list) -> None:
    """This process as rank ``rank`` of a world of ``world``: collectives, peer copies and barriers go to ``log``."""
    import torch.distributed._symmetric_memory as symm_mem

    def all_gather_into_tensor(out, inp, group=None):
        log.append(("all_gather_into_tensor", tuple(out.shape), tuple(inp.shape)))
        assert out.numel() == world * inp.numel()
        out.copy_(inp.reshape(1, -1).expand(world, -1).reshape(out.shape))

    def all_to_all_single(out, inp, group=None):
        log.append(("all_to_all_single", tuple(out.shape), tuple(inp.shape)))
        assert out.shape == inp.shape
        out.copy_(inp)

    def all_reduce(t, op=None, group=None):
        log.append(("all_reduce", tuple(t.shape), t.dtype))

    monkeypatch.setattr(par, "_group_world_rank", lambda group: (world, rank))
    monkeypatch.setattr(par.dist, "all_gather_into_tensor", all_gather_into_tensor)
    monkeypatch.setattr(par.dist, "all_to_all_single", all_to_all_single)
    monkeypatch.setattr(par.dist, "all_reduce", all_reduce)
    made = []
    monkeypatch.setattr(symm_mem, "empty", lambda shape, dtype, device: torch.zeros(shape, dtype=dtype))
    monkeypatch.setattr(symm_mem, "rendezvous",
                        lambda t, group: made.append(t) or Handle(world, rank, len(made) - 1, log))
