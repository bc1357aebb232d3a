"""Reduce-scatter and broadcast without a GPU: the header entry and binding of b2_reduce_scatter, its argument validation
through the library, Communicator.reduce_scatter_'s checks, and the torch.distributed-shaped helpers reduce_scatter_tensor,
reduce_scatter and broadcast on a stand-in communicator and with a process group up."""
import ctypes
import os
import re

import pytest
import torch
import torch.distributed as dist

from torchx_b200.ddp import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_reduce_scatter_and_the_binding_matches():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    decl = re.search(r"int\s+b2_reduce_scatter\(([^)]*)\);", src)
    assert decl, "b2_reduce_scatter is not declared"
    params = [p.strip() for p in decl.group(1).split(",")]
    assert params == ["b2_comm_t* comm", "void* out", "const void* in", "size_t n_elems", "int dtype", "int op", "void* stream"]
    assert re.search(r"b2_reduce_scatter\s+<- `dist.reduce_scatter_tensor` / `dist.reduce_scatter`", src)
    assert "b2_reduce_scatter" in N.SYMBOLS
    L = N.lib()
    fn = L.b2_reduce_scatter
    assert fn.restype is ctypes.c_int
    assert fn.argtypes == [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int,
                           ctypes.c_void_p]


def test_argument_validation_without_a_gpu():
    """In b2_allreduce_op's order: dtype, op, AVG on an integer dtype (even when empty), then n == 0 is a no-op, then the
    communicator.  Null buffers, overlaps and a poisoned communicator need one: tests/test_reduce_scatter_gpu.py."""
    L = N.lib()
    buf, other = ctypes.c_void_p(4096), ctypes.c_void_p(1 << 20)
    for dt in (-1, 5, 99):
        assert L.b2_reduce_scatter(None, buf, other, 8, dt, N.B2_OP_SUM, None) == N.B2_EINVAL, dt
        assert f"b2_reduce_scatter: unknown dtype {dt}".encode() in L.b2_last_error()
        assert L.b2_reduce_scatter(None, None, None, 0, dt, 42, None) == N.B2_EINVAL  # the dtype is checked first
        assert f"b2_reduce_scatter: unknown dtype {dt}".encode() in L.b2_last_error()
    for op in (-1, 4, 99):
        assert L.b2_reduce_scatter(None, buf, other, 8, N.B2_DT_FLOAT32, op, None) == N.B2_EINVAL, op
        assert f"b2_reduce_scatter: unknown op {op}".encode() in L.b2_last_error()
        assert L.b2_reduce_scatter(None, None, None, 0, N.B2_DT_INT32, op, None) == N.B2_EINVAL
    for dt, name in ((N.B2_DT_INT32, b"int32"), (N.B2_DT_INT64, b"int64")):
        for n in (8, 0):  # rejected even when empty
            assert L.b2_reduce_scatter(None, buf, other, n, dt, N.B2_OP_AVG, None) == N.B2_EINVAL
            assert b"b2_reduce_scatter: AVG needs a floating-point dtype, got " + name in L.b2_last_error()
    for dt in range(5):
        for op in range(4):
            if op == N.B2_OP_AVG and dt in (N.B2_DT_INT32, N.B2_DT_INT64):
                continue
            assert L.b2_reduce_scatter(None, None, None, 0, dt, op, None) == N.B2_OK, (dt, op)  # reads nothing else
            assert L.b2_reduce_scatter(None, buf, other, 8, dt, op, None) == N.B2_EINVAL, (dt, op)
            assert b"null communicator" in L.b2_last_error()


# ---- Communicator.reduce_scatter_ ------------------------------------------------------------------------------------
def _bare_communicator(world):
    """A Communicator whose checks run without a library handle (they all come before the call)."""
    from torchx_b200.ddp import Communicator

    c = Communicator.__new__(Communicator)
    c._h, c._owner, c.rank, c.world, c.device, c.ordered_stream = ctypes.c_void_p(), False, 0, world, 0, None
    return c


def test_communicator_checks_dtype_op_and_sizes():
    c = _bare_communicator(3)
    with pytest.raises(TypeError, match="reduce_scatter_: out is torch.int32, input is torch.int64"):
        c.reduce_scatter_(torch.zeros(2, dtype=torch.int32), torch.zeros(6, dtype=torch.int64))
    with pytest.raises(ValueError, match="input has 7 elements, needs 3 x 2"):
        c.reduce_scatter_(torch.zeros(2), torch.zeros(7))
    with pytest.raises(TypeError, match="reduce_scatter_: avg needs a floating-point tensor"):
        c.reduce_scatter_(torch.zeros(2, dtype=torch.int64), torch.zeros(6, dtype=torch.int64), "avg")
    with pytest.raises(TypeError, match="reduce_scatter_: unsupported dtype torch.float64"):
        c.reduce_scatter_(torch.zeros(2, dtype=torch.float64), torch.zeros(6, dtype=torch.float64))
    with pytest.raises(ValueError, match="reduce_scatter_: unsupported op 'product'"):
        c.reduce_scatter_(torch.zeros(2), torch.zeros(6), "product")
    with pytest.raises(ValueError, match="tensor on cpu"):  # the sizes fit: the device check is next
        c.reduce_scatter_(torch.zeros(2), torch.zeros(6))


# ---- the torch.distributed-shaped helpers ----------------------------------------------------------------------------
class _FakeComm:
    """Stands in for the native communicator: records calls; reduce_scatter_ writes block `rank` of its input plus 1000
    times the op's position in (sum, avg, min, max); broadcast_ adds 10 * root."""

    def __init__(self, world, rank=1):
        self.world, self.rank = world, rank
        self.calls = []

    def reduce_scatter_(self, out, t, op):
        self.calls.append(("reduce_scatter_", op, tuple(out.shape), tuple(t.shape), out.is_contiguous()))
        blk = t.reshape(self.world, -1)[self.rank]
        out.copy_((blk + 1000 * ("sum", "avg", "min", "max").index(op)).view(out.shape))
        return out

    def broadcast_(self, t, root=0):
        self.calls.append(("broadcast_", root))
        t.add_(10 * root)
        return t


def test_helpers_run_on_the_native_communicator(monkeypatch):
    import torchx_b200.distributed as D

    assert not dist.is_initialized()
    fake = _FakeComm(3)
    monkeypatch.setattr(D, "_COMM", fake)
    R = dist.ReduceOp
    inp = torch.arange(12, dtype=torch.int64).view(3, 4)
    out = torch.empty(4, dtype=torch.int64)
    assert D.reduce_scatter_tensor(out, inp) is None
    assert out.tolist() == [4, 5, 6, 7]
    D.reduce_scatter_tensor(out, inp, op=R.MAX, group=dist.group.WORLD)
    assert out.tolist() == [3004, 3005, 3006, 3007]
    x = torch.zeros(6)
    y = torch.empty(2)
    D.reduce_scatter_tensor(y, x, op=R.AVG)
    D.reduce_scatter_tensor(y, x, op=R(R.MIN))  # a ReduceOp instance, not only the enum value
    assert [c[1] for c in fake.calls] == ["sum", "max", "avg", "min"]

    # the list form: input_list[q] is block q, whatever its shape
    fake.calls.clear()
    lst = [torch.full((2, 2), q, dtype=torch.int32) for q in range(3)]
    o = torch.empty(2, 2, dtype=torch.int32)
    assert D.reduce_scatter(o, lst) is None
    assert o.tolist() == [[1, 1], [1, 1]]
    assert fake.calls == [("reduce_scatter_", "sum", (2, 2), (12,), True)]
    # input_list tensors of any layout: flattened in their element order, block q = input_list[q]
    D.reduce_scatter(o, [(torch.arange(4, dtype=torch.int32).view(2, 2) * (q + 1)).t() for q in range(3)], op=R.MIN)
    assert o.tolist() == [[2000, 2004], [2002, 2006]]

    # broadcast
    s = torch.tensor([5, 6])
    assert D.broadcast(s, src=2) is None
    assert s.tolist() == [25, 26] and fake.calls[-1] == ("broadcast_", 2)
    D.broadcast(s, 0, group=dist.group.WORLD)
    assert fake.calls[-1] == ("broadcast_", 0)


def test_helpers_refuse_what_the_fabric_does_not_have(monkeypatch):
    import torchx_b200.distributed as D

    fake = _FakeComm(3)
    monkeypatch.setattr(D, "_COMM", fake)
    R = dist.ReduceOp
    out, inp = torch.empty(4), torch.zeros(12)
    lst = [torch.zeros(4) for _ in range(3)]
    for call in (lambda: D.reduce_scatter_tensor(out, inp, async_op=True), lambda: D.reduce_scatter(out, lst, async_op=True),
                 lambda: D.broadcast(out, 0, async_op=True)):
        with pytest.raises(NotImplementedError, match="no work handles"):
            call()
    for call in (lambda: D.reduce_scatter_tensor(out, inp, group=object()), lambda: D.reduce_scatter(out, lst, group=object()),
                 lambda: D.broadcast(out, 0, group=object())):
        with pytest.raises(NotImplementedError, match="no subgroups"):
            call()
    for o in (R.PRODUCT, R.BAND, R.BOR, R.BXOR):
        for call in (lambda: D.reduce_scatter_tensor(out, inp, op=o), lambda: D.reduce_scatter(out, lst, op=o)):
            with pytest.raises(ValueError, match="supports SUM, AVG, MIN and MAX"):
                call()
    with pytest.raises(ValueError, match="input_list has 2 tensors, world size is 3"):
        D.reduce_scatter(out, lst[:2])
    with pytest.raises(ValueError, match="every tensor of input_list must be torch.float32 with 4 elements"):
        D.reduce_scatter(out, [torch.zeros(4), torch.zeros(5), torch.zeros(4)])
    with pytest.raises(ValueError, match="every tensor of input_list"):
        D.reduce_scatter(out, [torch.zeros(4), torch.zeros(4, dtype=torch.int32), torch.zeros(4)])
    assert fake.calls == []  # nothing reached the communicator


def test_helpers_delegate_to_torch_distributed_with_a_process_group(monkeypatch):
    """A process group is up (even with a native communicator next to it): torch.distributed's own functions run, with
    their own rules - async work handles, subgroups and PRODUCT included."""
    import torchx_b200.distributed as D

    fake = _FakeComm(2)
    monkeypatch.setattr(D, "_COMM", fake)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    seen = []
    monkeypatch.setattr(dist, "reduce_scatter_tensor",
                        lambda o, i, op, group, async_op: seen.append(("reduce_scatter_tensor", op, group, async_op)) or "w1")
    monkeypatch.setattr(dist, "reduce_scatter",
                        lambda o, lst, op, group, async_op: seen.append(("reduce_scatter", len(lst), op, async_op)) or "w2")
    monkeypatch.setattr(dist, "broadcast", lambda t, src, group, async_op: seen.append(("broadcast", src, async_op)) or "w3")
    g = object()
    t = torch.zeros(2)
    assert D.reduce_scatter_tensor(t, torch.zeros(4), op=dist.ReduceOp.PRODUCT, group=g, async_op=True) == "w1"
    assert D.reduce_scatter(t, [t, t, t], async_op=True) == "w2"
    assert D.broadcast(t, src=1, async_op=True) == "w3"
    assert seen == [("reduce_scatter_tensor", dist.ReduceOp.PRODUCT, g, True), ("reduce_scatter", 3, dist.ReduceOp.SUM, True),
                    ("broadcast", 1, True)]
    assert fake.calls == []


def test_helpers_delegate_without_the_native_communicator(monkeypatch):
    import torchx_b200.distributed as D

    monkeypatch.setattr(D, "_COMM", None)
    seen = []
    monkeypatch.setattr(dist, "reduce_scatter_tensor", lambda *a, **k: seen.append("reduce_scatter_tensor"))
    monkeypatch.setattr(dist, "reduce_scatter", lambda *a, **k: seen.append("reduce_scatter"))
    monkeypatch.setattr(dist, "broadcast", lambda *a, **k: seen.append("broadcast"))
    t = torch.zeros(2)
    D.reduce_scatter_tensor(t, torch.zeros(4))
    D.reduce_scatter(t, [t, t])
    D.broadcast(t, 0)
    assert seen == ["reduce_scatter_tensor", "reduce_scatter", "broadcast"]
