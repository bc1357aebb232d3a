"""Point-to-point without a GPU: the header entries and bindings of b2_p2p / b2_p2p_eager_bytes, the checks that come before
the communicator is read, Communicator.p2p_'s argument checks, and the torch.distributed-shaped helpers send, recv, isend,
irecv, P2POp, batch_isend_irecv, gather and scatter on a stand-in communicator and with a process group up.  The checks
that need a communicator: tests/test_p2p_gpu.py."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.distributed as dist

from torchx_b200.ddp import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_p2p_and_the_binding_matches():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    decl = re.search(r"int\s+b2_p2p\(([^)]*)\);", src)
    assert decl, "b2_p2p is not declared"
    params = [" ".join(p.split()) for p in decl.group(1).split(",")]
    assert params == ["b2_comm_t* comm", "const b2_p2p_op_t* ops", "int n_ops", "void* stream"]
    assert re.search(r"size_t\s+b2_p2p_eager_bytes\(const b2_comm_t\* comm\);", src)
    assert re.search(r"#define B2_P2P_MAX_OPS 64\b", src) and N.B2_P2P_MAX_OPS == 64
    struct = re.search(r"typedef struct b2_p2p_op \{(.*?)\} b2_p2p_op_t;", src, re.S).group(1)
    fields = [" ".join(re.sub(r"/\*.*?\*/", "", f).split()) for f in struct.split(";") if re.sub(r"/\*.*?\*/", "", f).strip()]
    assert fields == ["int peer", "int is_send", "void* ptr", "size_t bytes"]
    assert [f[0] for f in N.B2P2pOp._fields_] == ["peer", "is_send", "ptr", "bytes"]
    assert ctypes.sizeof(N.B2P2pOp) == 24
    assert "b2_p2p             <- dist.send / dist.recv / dist.batch_isend_irecv" in src
    assert {"b2_p2p", "b2_p2p_eager_bytes"} <= set(N.SYMBOLS)
    L = N.lib()
    assert L.b2_p2p.restype is ctypes.c_int
    assert L.b2_p2p.argtypes == [ctypes.c_void_p, ctypes.POINTER(N.B2P2pOp), ctypes.c_int, ctypes.c_void_p]
    assert L.b2_p2p_eager_bytes.restype is ctypes.c_size_t and L.b2_p2p_eager_bytes.argtypes == [ctypes.c_void_p]


def test_argument_validation_without_a_gpu():
    """A null communicator comes first; nothing else is read before it."""
    L = N.lib()
    ops = (N.B2P2pOp * 1)(N.B2P2pOp(1, 1, 4096, 16))
    assert L.b2_p2p(None, ops, 1, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"null communicator"
    assert L.b2_p2p(None, None, 0, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"null communicator"
    assert L.b2_p2p_eager_bytes(None) == 0


# ---- Communicator.p2p_ -----------------------------------------------------------------------------------------------
def _bare_communicator(world, rank=0):
    """A Communicator whose checks run without a library handle (they all come before the call)."""
    from torchx_b200.ddp import Communicator

    c = Communicator.__new__(Communicator)
    c._h, c._owner, c.rank, c.world, c.device, c.ordered_stream = ctypes.c_void_p(), False, rank, world, 0, None
    return c


def test_communicator_checks_ops_peers_and_tensors():
    c = _bare_communicator(3, rank=1)
    t = torch.zeros(2)
    with pytest.raises(ValueError, match=r"p2p_: needs 1\.\.64 ops, got 0"):
        c.p2p_([])
    with pytest.raises(ValueError, match=r"p2p_: needs 1\.\.64 ops, got 65"):
        c.p2p_([("send", t, 0)] * 65)
    with pytest.raises(ValueError, match="p2p_: op 0 is 'put', not 'send' or 'recv'"):
        c.p2p_([("put", t, 0)])
    for k, peer in enumerate((1, 3, -1, None, 0.0, True, np.int64(1))):  # self, out of range, not a rank
        with pytest.raises(ValueError, match=f"p2p_: op 1 names peer {re.escape(repr(peer))}; rank 1 of 3 can only name another rank"):
            c.p2p_([("send", t, 0), ("recv", t, peer)])
    for peer in (2, np.int64(2), np.int32(0)):  # integers as torch takes them reach the next check: the wrong device
        with pytest.raises(ValueError, match="tensor on cpu, communicator on cuda:0"):
            c.p2p_([("send", t, peer)])
    # the contiguity check comes after the device check: tests/test_p2p_gpu.py
    c1 = _bare_communicator(1)
    with pytest.raises(ValueError, match="rank 0 of 1 can only name another rank"):
        c1.p2p_([("send", t, 0)])


# ---- the torch.distributed-shaped helpers ----------------------------------------------------------------------------
class _FakeComm:
    """Stands in for the native communicator: records every p2p_ batch as (kind, data_ptr, shape, peer) tuples."""

    def __init__(self, world, rank=0):
        self.world, self.rank, self.device = world, rank, 0
        self.calls = []

    def p2p_(self, ops, stream=None):
        self.calls.append([(kind, t.data_ptr(), tuple(t.shape), peer) for kind, t, peer in ops])


class _FakeEvent:
    def __init__(self):
        self.recorded = 0

    def record(self, stream=None):
        self.recorded += 1

    def query(self):
        return self.recorded > 0


@pytest.fixture
def fabric(monkeypatch):
    """A stand-in communicator of `world` ranks with this rank `rank`, and CUDA events / streams that need no GPU."""
    import torchx_b200.distributed as D

    assert not dist.is_initialized()
    monkeypatch.setattr(torch.cuda, "Event", _FakeEvent)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: None)

    def make(world, rank=0):
        fake = _FakeComm(world, rank)
        monkeypatch.setattr(D, "_COMM", fake)
        return D, fake

    return make


def test_send_recv_isend_irecv_are_batches_of_one(fabric):
    D, fake = fabric(3, rank=1)
    a, b = torch.zeros(4), torch.zeros(2, 3, dtype=torch.int64)
    assert D.send(a, 2) is None
    assert D.recv(b, 0, tag=7) == 0
    w1 = D.isend(b, 0, group=dist.group.WORLD)
    w2 = D.irecv(a, 2)
    assert fake.calls == [[("send", a.data_ptr(), (4,), 2)], [("recv", b.data_ptr(), (2, 3), 0)],
                          [("send", b.data_ptr(), (2, 3), 0)], [("recv", a.data_ptr(), (4,), 2)]]
    assert w1.wait() is True and w2.wait() is True
    assert w1.is_completed() and w2.is_completed()


def test_p2pop_is_a_record_without_a_process_group(fabric):
    D, fake = fabric(4, rank=2)
    x, y, z = torch.zeros(3), torch.ones(5), torch.zeros(1, dtype=torch.uint8)
    ops = [D.P2POp(D.isend, x, 3), D.P2POp(dist.irecv, y, 1, tag=4), D.P2POp(dist.isend, z, 0), D.P2POp(D.irecv, x, 3)]
    assert isinstance(ops[0], D.P2POp) and ops[1].peer == 1 and ops[1].tag == 4 and ops[2].tensor is z
    works = D.batch_isend_irecv(ops)
    assert fake.calls == [[("send", x.data_ptr(), (3,), 3), ("recv", y.data_ptr(), (5,), 1), ("send", z.data_ptr(), (1,), 0),
                           ("recv", x.data_ptr(), (3,), 3)]]
    assert len(works) == 4 and all(w.wait() and w.is_completed() for w in works)
    with pytest.raises(ValueError, match="Invalid ``op``"):
        D.P2POp(D.send, x, 3)


def test_batch_isend_irecv_refuses_what_it_cannot_run_in_one_launch(fabric):
    D, fake = fabric(2, rank=0)
    t = torch.zeros(1)
    with pytest.raises(ValueError, match="batch_isend_irecv: 65 ops, the b200 communicator takes at most 64 in one batch"):
        D.batch_isend_irecv([D.P2POp(D.isend, t, 1)] * 65)
    with pytest.raises(ValueError, match="p2p_op_list is empty"):
        D.batch_isend_irecv([])
    with pytest.raises(NotImplementedError, match="no subgroups"):
        D.batch_isend_irecv([D.P2POp(D.isend, t, 1), D.P2POp(D.irecv, t, 1, group=object())])
    assert fake.calls == []
    D.batch_isend_irecv([D.P2POp(D.isend, t, 1)] * 64)
    assert len(fake.calls) == 1 and len(fake.calls[0]) == 64


@pytest.mark.parametrize("world", [1, 2, 4])
def test_gather_root_receives_in_one_batch_and_others_send(fabric, world):
    for dst in range(world):
        for rank in range(world):
            D, fake = fabric(world, rank)
            t = torch.full((2, 2), float(rank))
            if rank == dst:
                lst = [torch.zeros(2, 2) for _ in range(world)]
                assert D.gather(t, lst, dst=dst) is None
                want = [[("recv", lst[r].data_ptr(), (2, 2), r) for r in range(world) if r != dst]] if world > 1 else []
                assert fake.calls == want
                assert torch.equal(lst[dst], t)  # the own block is a local copy
            else:
                assert D.gather(t, None, dst=dst) is None
                assert fake.calls == [[("send", t.data_ptr(), (2, 2), dst)]]


@pytest.mark.parametrize("world", [1, 2, 4])
def test_scatter_root_sends_in_one_batch_and_others_receive(fabric, world):
    for src in range(world):
        for rank in range(world):
            D, fake = fabric(world, rank)
            t = torch.zeros(3, dtype=torch.int32)
            if rank == src:
                lst = [torch.full((3,), r, dtype=torch.int32) for r in range(world)]
                assert D.scatter(t, lst, src=src) is None
                want = [[("send", lst[r].data_ptr(), (3,), r) for r in range(world) if r != src]] if world > 1 else []
                assert fake.calls == want
                assert t.tolist() == [src] * 3
            else:
                assert D.scatter(t, [], src=src) is None
                assert fake.calls == [[("recv", t.data_ptr(), (3,), src)]]


def test_gather_and_scatter_check_their_arguments(fabric):
    D, fake = fabric(3, rank=1)
    t = torch.zeros(2)
    with pytest.raises(ValueError, match="must NOT be specified on non-destination ranks"):
        D.gather(t, [t, t, t], dst=0)
    with pytest.raises(ValueError, match="must be specified on destination rank"):
        D.gather(t, None, dst=1)
    with pytest.raises(ValueError, match="gather: gather_list has 2 tensors, world size is 3"):
        D.gather(t, [t, t], dst=1)
    with pytest.raises(ValueError, match="gather: gather_list: every tensor must be torch.float32 with 2 elements"):
        D.gather(t, [t, torch.zeros(3), t], dst=1)
    with pytest.raises(ValueError, match="gather: dst 3 is not a rank of a world of 3"):
        D.gather(t, None, dst=3)
    with pytest.raises(ValueError, match="must NOT be specified on non-source ranks"):
        D.scatter(t, [t, t, t], src=2)
    with pytest.raises(ValueError, match="must be specified on source rank"):
        D.scatter(t, None, src=1)
    with pytest.raises(ValueError, match="scatter: scatter_list: every tensor must be torch.float32 with 2 elements"):
        D.scatter(t, [t, t, torch.zeros(2, dtype=torch.int64)], src=1)
    with pytest.raises(ValueError, match="scatter: src -1 is not a rank"):
        D.scatter(t, None, src=-1)
    assert fake.calls == []


def test_helpers_refuse_what_the_fabric_does_not_have(fabric):
    D, fake = fabric(2, rank=0)
    t, lst = torch.zeros(4), [torch.zeros(4), torch.zeros(4)]
    for call in (lambda: D.recv(t), lambda: D.irecv(t), lambda: D.batch_isend_irecv([D.P2POp(D.irecv, t, None)])):
        with pytest.raises(NotImplementedError, match="cannot receive from any source"):
            call()
    for call in (lambda: D.gather(t, lst, async_op=True), lambda: D.scatter(t, lst, async_op=True)):
        with pytest.raises(NotImplementedError, match="no work handles"):
            call()
    g = object()
    for call in (lambda: D.send(t, 1, group=g), lambda: D.recv(t, 1, group=g), lambda: D.isend(t, 1, group=g),
                 lambda: D.irecv(t, 1, group=g), lambda: D.gather(t, lst, group=g), lambda: D.scatter(t, lst, group=g)):
        with pytest.raises(NotImplementedError, match="no subgroups"):
            call()
    assert fake.calls == []


def test_helpers_delegate_to_torch_distributed_with_a_process_group(monkeypatch):
    """A process group is up (even with a native communicator next to it): torch.distributed's own functions run, with
    their own rules - any-source receives, work handles and subgroups included.  (Stand-ins here; P2POp and
    batch_isend_irecv under a real group: the gloo tests below.)"""
    import torchx_b200.distributed as D

    fake = _FakeComm(2)
    monkeypatch.setattr(D, "_COMM", fake)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    seen = []
    monkeypatch.setattr(dist, "send", lambda t, dst, group, tag: seen.append(("send", dst, group, tag)))
    monkeypatch.setattr(dist, "recv", lambda t, src, group, tag: seen.append(("recv", src, group, tag)) or 5)
    monkeypatch.setattr(dist, "isend", lambda t, dst, group, tag: seen.append(("isend", dst, group, tag)) or "w1")
    monkeypatch.setattr(dist, "irecv", lambda t, src, group, tag: seen.append(("irecv", src, group, tag)) or "w2")
    monkeypatch.setattr(dist, "batch_isend_irecv", lambda lst: seen.append(("batch", lst)) or ["w3"])
    monkeypatch.setattr(dist, "gather", lambda t, lst, dst, group, async_op: seen.append(("gather", dst, group, async_op)) or "w4")
    monkeypatch.setattr(dist, "scatter", lambda t, lst, src, group, async_op: seen.append(("scatter", src, group, async_op)) or "w5")
    g, t = object(), torch.zeros(2)
    D.send(t, 1, group=g, tag=3)
    assert D.recv(t, group=g) == 5
    assert D.isend(t, 1, tag=2) == "w1" and D.irecv(t) == "w2"
    op = object()  # P2POp itself with a real process group: test_p2pop_and_batch_under_a_real_gloo_group
    assert D.batch_isend_irecv([op]) == ["w3"]
    assert D.gather(t, None, dst=1, group=g, async_op=True) == "w4"
    assert D.scatter(t, None, src=1, async_op=True) == "w5"
    assert seen == [("send", 1, g, 3), ("recv", None, g, 0), ("isend", 1, None, 2), ("irecv", None, None, 0), ("batch", [op]),
                    ("gather", 1, g, True), ("scatter", 1, None, True)]
    assert fake.calls == []


def test_helpers_delegate_without_the_native_communicator(monkeypatch):
    import torchx_b200.distributed as D

    monkeypatch.setattr(D, "_COMM", None)
    seen = []
    for name in ("send", "recv", "isend", "irecv", "P2POp", "batch_isend_irecv", "gather", "scatter"):
        monkeypatch.setattr(dist, name, lambda *a, _n=name, **k: seen.append(_n))
    t = torch.zeros(2)
    D.send(t, 1)
    D.recv(t, 1)
    D.isend(t, 1)
    D.irecv(t)
    D.P2POp(D.isend, t, 1)
    D.batch_isend_irecv([])
    D.gather(t)
    D.scatter(t)
    assert seen == ["send", "recv", "isend", "irecv", "P2POp", "batch_isend_irecv", "gather", "scatter"]


# ---- under a real torch.distributed process group (gloo, CPU) ---------------------------------------------------------
def test_p2pop_under_a_real_one_rank_gloo_group(tmp_path, monkeypatch):
    """With a process group up, P2POp is torch's own, and this module's isend / irecv become torch's: torch.distributed's
    P2POp accepts nothing else."""
    import torchx_b200.distributed as D

    monkeypatch.setattr(D, "_COMM", None)
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1)
    try:
        t = torch.zeros(3)
        ops = [D.P2POp(D.isend, t, 0), D.P2POp(D.irecv, t, 0, tag=5), D.P2POp(dist.isend, t, 0)]
        assert all(type(p) is dist.P2POp for p in ops)
        assert [p.op for p in ops] == [dist.isend, dist.irecv, dist.isend] and ops[1].tag == 5
        with pytest.raises(ValueError, match="Invalid ``op``"):
            D.P2POp(D.send, t, 0)
    finally:
        dist.destroy_process_group()


def _gloo_rank(rank, store, out):
    """One rank of a two-process gloo group running a script written for either backend."""
    import torchx_b200.distributed as D

    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=2)
    try:
        peer = 1 - rank
        mine = torch.arange(5, dtype=torch.float64) + 10 * rank
        got = torch.zeros(5, dtype=torch.float64)
        for w in D.batch_isend_irecv([D.P2POp(D.isend, mine, peer), D.P2POp(D.irecv, got, peer)]):
            w.wait()
        one = torch.zeros(2, dtype=torch.int64)
        if rank == 0:
            D.send(torch.tensor([7, 8]), 1)
        else:
            assert D.recv(one, 0) == 0
        torch.save({"got": got, "one": one}, out)
    finally:
        dist.destroy_process_group()


def test_batch_isend_irecv_under_a_real_two_rank_gloo_group(tmp_path):
    import multiprocessing as mp

    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_gloo_rank, args=(r, str(tmp_path / "store"), str(tmp_path / f"r{r}.pt"))) for r in range(2)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(120)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    assert [p.exitcode for p in procs] == [0, 0]
    r0, r1 = (torch.load(tmp_path / f"r{r}.pt") for r in range(2))
    assert r0["got"].tolist() == [10.0, 11.0, 12.0, 13.0, 14.0] and r1["got"].tolist() == [0.0, 1.0, 2.0, 3.0, 4.0]
    assert r1["one"].tolist() == [7, 8]
