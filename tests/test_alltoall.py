"""All-to-all without a GPU: the header entries and bindings of b2_alltoall / b2_alltoall_max_bytes, the checks that come
before the communicator is read, Communicator.alltoall_'s argument checks, and the torch.distributed-shaped helpers
all_to_all_single and all_to_all on a stand-in communicator and with a process group up.  Null pointers with a count,
overlaps and a poisoned communicator need a communicator: tests/test_alltoall_gpu.py."""
import ctypes
import os
import re

import pytest
import torch
import torch.distributed as dist

from torchx_b200.ddp import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_alltoall_and_the_binding_matches():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    decl = re.search(r"int\s+b2_alltoall\(([^)]*)\);", src)
    assert decl, "b2_alltoall is not declared"
    params = [" ".join(p.split()) for p in decl.group(1).split(",")]
    assert params == ["b2_comm_t* comm", "void* const* out", "const size_t* recv_bytes", "const void* const* in",
                      "const size_t* send_bytes", "void* stream"]
    assert re.search(r"size_t\s+b2_alltoall_max_bytes\(const b2_comm_t\* comm\);", src)
    assert re.search(r"b2_alltoall, b2_alltoall_max_bytes <- `dist.all_to_all_single` / `dist.all_to_all`", src)
    assert {"b2_alltoall", "b2_alltoall_max_bytes"} <= set(N.SYMBOLS)
    L = N.lib()
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    assert L.b2_alltoall.restype is ctypes.c_int
    assert L.b2_alltoall.argtypes == [vp, ctypes.POINTER(vp), ctypes.POINTER(sz), ctypes.POINTER(vp), ctypes.POINTER(sz), vp]
    assert L.b2_alltoall_max_bytes.restype is sz and L.b2_alltoall_max_bytes.argtypes == [vp]


def test_argument_validation_without_a_gpu():
    """A null communicator first, then null arrays; nothing else is read before the communicator."""
    L = N.lib()
    ptrs, sizes = (ctypes.c_void_p * 2)(4096, 8192), (ctypes.c_size_t * 2)(16, 16)
    assert L.b2_alltoall(None, ptrs, sizes, ptrs, sizes, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"null communicator"
    assert L.b2_alltoall(None, None, None, None, None, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"null communicator"
    assert L.b2_alltoall_max_bytes(None) == 0


# ---- Communicator.alltoall_ ------------------------------------------------------------------------------------------
def _bare_communicator(world):
    """A Communicator whose checks run without a library handle (they all come before the call)."""
    from torchx_b200.ddp import Communicator

    c = Communicator.__new__(Communicator)
    c._h, c._owner, c.rank, c.world, c.device, c.ordered_stream = ctypes.c_void_p(), False, 0, world, 0, None
    return c


def test_communicator_checks_lengths_and_dtypes():
    c = _bare_communicator(3)
    z = [torch.zeros(2) for _ in range(3)]
    with pytest.raises(ValueError, match="alltoall_: needs 3 output and 3 input tensors, got 2 and 3"):
        c.alltoall_(z[:2], z)
    with pytest.raises(ValueError, match="needs 3 output and 3 input tensors, got 3 and 4"):
        c.alltoall_(z, z + [torch.zeros(2)])
    with pytest.raises(TypeError, match=r"alltoall_: every tensor must have one dtype, got \['torch.float32', 'torch.int64'\]"):
        c.alltoall_(z, z[:2] + [torch.zeros(2, dtype=torch.int64)])
    with pytest.raises(TypeError, match="one dtype"):
        c.alltoall_([torch.zeros(2, dtype=torch.bfloat16)] + z[1:], z)
    # any dtype is accepted: the device check is next (the contiguity check after it: tests/test_alltoall_gpu.py)
    with pytest.raises(ValueError, match="tensor on cpu"):
        c.alltoall_([torch.zeros(2, dtype=torch.complex64)] * 3, [torch.zeros(2, dtype=torch.complex64)] * 3)


# ---- the torch.distributed-shaped helpers ----------------------------------------------------------------------------
class _FakeComm:
    """Stands in for the native communicator: records the address and shape of every tensor alltoall_ was given, and
    copies ins[q] into outs[q] where their shapes agree (the exchange of a world whose every rank holds this rank's
    data)."""

    def __init__(self, world, rank=1):
        self.world, self.rank = world, rank
        self.calls = []

    def alltoall_(self, outs, ins):
        self.calls.append(([(t.data_ptr(), tuple(t.shape)) for t in outs], [(t.data_ptr(), tuple(t.shape)) for t in ins]))
        for o, i in zip(outs, ins):
            if o.shape == i.shape:
                o.copy_(i)
        return outs


def test_all_to_all_single_passes_views_of_its_tensors(monkeypatch):
    import torchx_b200.distributed as D

    assert not dist.is_initialized()
    fake = _FakeComm(3)
    monkeypatch.setattr(D, "_COMM", fake)
    # even split: 6 rows of 2 -> 3 blocks of 2 rows
    inp = torch.arange(12, dtype=torch.int64).view(6, 2)
    out = torch.zeros(6, 2, dtype=torch.int64)
    assert D.all_to_all_single(out, inp) is None
    (outs, ins), = fake.calls
    row = 2 * 8  # bytes of one row
    assert outs == [(out.data_ptr() + 2 * k * row, (2, 2)) for k in range(3)]
    assert ins == [(inp.data_ptr() + 2 * k * row, (2, 2)) for k in range(3)]
    assert torch.equal(out, inp)
    # uneven splits on both sides, empty blocks included; [] means even, as in torch
    fake.calls.clear()
    x = torch.arange(5, dtype=torch.float32)
    y = torch.zeros(7)
    D.all_to_all_single(y, x, output_split_sizes=[3, 0, 4], input_split_sizes=[1, 4, 0], group=dist.group.WORLD)
    (outs, ins), = fake.calls
    assert outs == [(y.data_ptr(), (3,)), (0, (0,)), (y.data_ptr() + 12, (4,))]  # an empty view has no address
    assert ins == [(x.data_ptr(), (1,)), (x.data_ptr() + 4, (4,)), (0, (0,))]
    fake.calls.clear()
    D.all_to_all_single(torch.zeros(3, 4), torch.zeros(6, 4), output_split_sizes=[], input_split_sizes=(2, 2, 2))
    (outs, ins), = fake.calls
    assert [s for _, s in outs] == [(1, 4)] * 3 and [s for _, s in ins] == [(2, 4)] * 3


def test_all_to_all_single_rejects_bad_splits(monkeypatch):
    import torchx_b200.distributed as D

    fake = _FakeComm(3)
    monkeypatch.setattr(D, "_COMM", fake)
    with pytest.raises(ValueError, match="all_to_all_single: input has 7 rows, not a multiple of the world size 3"):
        D.all_to_all_single(torch.zeros(6), torch.zeros(7))
    with pytest.raises(ValueError, match="all_to_all_single: output has 5 rows, not a multiple of the world size 3"):
        D.all_to_all_single(torch.zeros(5), torch.zeros(6))
    bad = {"sum": [1, 2, 2], "length": [3, 3], "negative": [4, -1, 3]}
    for what, sizes in bad.items():
        with pytest.raises(ValueError, match=r"input_split_sizes .* must be 3 row counts >= 0 summing to the 6 rows of input"):
            D.all_to_all_single(torch.zeros(6), torch.zeros(6), input_split_sizes=sizes)
        with pytest.raises(ValueError, match=r"output_split_sizes .* summing to the 6 rows of output"):
            D.all_to_all_single(torch.zeros(6), torch.zeros(6), output_split_sizes=sizes)
    assert fake.calls == []


def test_all_to_all_passes_the_lists_as_they_are(monkeypatch):
    import torchx_b200.distributed as D

    fake = _FakeComm(2)
    monkeypatch.setattr(D, "_COMM", fake)
    outs = [torch.zeros(3, dtype=torch.int32), torch.zeros(2, 2, dtype=torch.int32)]
    ins = [torch.arange(3, dtype=torch.int32), torch.ones(2, 2, dtype=torch.int32)]
    assert D.all_to_all(outs, ins) is None
    assert fake.calls == [([(t.data_ptr(), tuple(t.shape)) for t in outs], [(t.data_ptr(), tuple(t.shape)) for t in ins])]
    assert outs[0].tolist() == [0, 1, 2] and outs[1].tolist() == [[1, 1], [1, 1]]


def test_helpers_refuse_what_the_fabric_does_not_have(monkeypatch):
    import torchx_b200.distributed as D

    fake = _FakeComm(2)
    monkeypatch.setattr(D, "_COMM", fake)
    t, lst = torch.zeros(4), [torch.zeros(2), torch.zeros(2)]
    for call in (lambda: D.all_to_all_single(t, t, async_op=True), lambda: D.all_to_all(lst, lst, async_op=True)):
        with pytest.raises(NotImplementedError, match="no work handles"):
            call()
    for call in (lambda: D.all_to_all_single(t, t, group=object()), lambda: D.all_to_all(lst, lst, group=object())):
        with pytest.raises(NotImplementedError, match="no subgroups"):
            call()
    assert fake.calls == []


def test_helpers_delegate_to_torch_distributed_with_a_process_group(monkeypatch):
    """A process group is up (even with a native communicator next to it): torch.distributed's own functions run, with
    their own rules - async work handles and subgroups included."""
    import torchx_b200.distributed as D

    fake = _FakeComm(2)
    monkeypatch.setattr(D, "_COMM", fake)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    seen = []
    monkeypatch.setattr(dist, "all_to_all_single",
                        lambda o, i, output_split_sizes, input_split_sizes, group, async_op:
                        seen.append(("all_to_all_single", output_split_sizes, input_split_sizes, group, async_op)) or "w1")
    monkeypatch.setattr(dist, "all_to_all", lambda o, i, group, async_op: seen.append(("all_to_all", len(o), group, async_op)) or "w2")
    g = object()
    t = torch.zeros(4)
    assert D.all_to_all_single(t, t, [1, 3], [2, 2], group=g, async_op=True) == "w1"
    assert D.all_to_all([t, t, t], [t, t, t], async_op=True) == "w2"
    assert seen == [("all_to_all_single", [1, 3], [2, 2], g, True), ("all_to_all", 3, None, True)]
    assert fake.calls == []


def test_helpers_delegate_without_the_native_communicator(monkeypatch):
    import torchx_b200.distributed as D

    monkeypatch.setattr(D, "_COMM", None)
    seen = []
    monkeypatch.setattr(dist, "all_to_all_single", lambda *a, **k: seen.append("all_to_all_single"))
    monkeypatch.setattr(dist, "all_to_all", lambda *a, **k: seen.append("all_to_all"))
    t = torch.zeros(2)
    D.all_to_all_single(t, t)
    D.all_to_all([t], [t])
    assert seen == ["all_to_all_single", "all_to_all"]
