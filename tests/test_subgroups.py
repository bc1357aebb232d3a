"""Process subgroups without a GPU: b2_comm_create_group's binding and the checks that come before a communicator is read,
B200Group's rank translation, every torchx_b200.distributed helper with a B200Group on stand-in communicators (global and
group ranks, ranks outside the group, calls from a non-member), new_group / new_subgroups*, SyncBatchNorm on a stand-in
group, and the refusal of any other group object.  On the GPU: tests/test_subgroups_gpu.py."""
import ctypes
import os
import re
import warnings

import pytest
import torch
import torch.distributed as dist

from torchx_b200.ddp import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_create_group_and_the_binding_matches():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    decl = re.search(r"int\s+b2_comm_create_group\(([^)]*)\);", src)
    params = [" ".join(p.split()) for p in decl.group(1).split(",")]
    assert params == ["b2_comm_t** out", "const b2_comm_t* parent", "int n_ranks", "const int* ranks", "size_t stage_bytes"]
    assert int(re.search(r"#define B2_GROUP_STAGE_MB (\d+)", src).group(1)) == N.B2_GROUP_STAGE_MB
    assert "b2_comm_create_group" in re.search(r"#define B2_ABI_VERSION 3 /\*(.*?)\*/", src, re.S).group(1)
    L = N.lib()
    assert L.b2_comm_create_group.restype is ctypes.c_int
    assert L.b2_comm_create_group.argtypes == [ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p, ctypes.c_int,
                                               ctypes.POINTER(ctypes.c_int), ctypes.c_size_t]


def test_argument_validation_without_a_gpu():
    L = N.lib()
    out = ctypes.c_void_p(1234)
    ranks = (ctypes.c_int * 2)(0, 1)
    assert L.b2_comm_create_group(None, None, 2, ranks, 0) == N.B2_EINVAL
    assert L.b2_last_error() == b"b2_comm_create_group: null out"
    assert L.b2_comm_create_group(ctypes.byref(out), None, 2, ranks, 0) == N.B2_EINVAL
    assert L.b2_last_error() == b"b2_comm_create_group: null parent"
    assert out.value is None  # *out is cleared before anything else is checked


# ---- B200Group -------------------------------------------------------------------------------------------------------
class _FakeComm:
    """Stands in for a native communicator: records every call as (method, args) with tensors as data pointers."""

    def __init__(self, world, rank=0):
        self.world, self.rank, self.device, self.ordered_stream = world, rank, 0, None
        self.calls = []

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)

        def call(*args, **kw):
            self.calls.append((name, args, kw))
        return call


def _group(D, ranks, me):
    return D.B200Group(_FakeComm(len(ranks), ranks.index(me)), ranks)


@pytest.fixture
def fabric(monkeypatch):
    import torchx_b200.distributed as D

    assert not dist.is_initialized()
    monkeypatch.setattr(torch.cuda, "Event", lambda: type("E", (), {"record": lambda s, st=None: None, "query": lambda s: True})())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: None)

    def make(world, rank):
        world_comm = _FakeComm(world, rank)
        monkeypatch.setattr(D, "_COMM", world_comm)
        return D, world_comm

    return make


def test_group_rank_translation(fabric):
    D, _ = fabric(8, 5)
    g = _group(D, [1, 3, 5, 6], 5)
    assert (g.rank(), g.size(), g.ranks) == (2, 4, [1, 3, 5, 6])
    assert [g.get_group_rank(r) for r in (1, 3, 5, 6)] == [0, 1, 2, 3]
    assert [g.get_global_rank(r) for r in range(4)] == [1, 3, 5, 6]
    for bad in (0, 2, 7, 8, -1, None, 1.0, True):
        with pytest.raises(ValueError, match="is not part of group"):
            g.get_group_rank(bad)
    for bad in (4, -1, None):
        with pytest.raises(ValueError, match="is not part of group"):
            g.get_global_rank(bad)


def test_collectives_run_on_the_group_communicator(fabric):
    D, world = fabric(4, 2)
    g = _group(D, [0, 2, 3], 2)
    t, lst = torch.zeros(6), [torch.zeros(2) for _ in range(3)]
    D.all_reduce(t, op=dist.ReduceOp.MAX, group=g)
    D.all_gather_into_tensor(torch.zeros(18), t, group=g)
    D.all_gather(lst, torch.zeros(2), group=g)
    D.reduce_scatter_tensor(torch.zeros(2), t, group=g)
    D.reduce_scatter(torch.zeros(2), lst, group=g)
    D.all_to_all_single(torch.zeros(6), t, group=g)
    D.all_to_all(lst, lst, group=g)
    names = [c[0] for c in g.comm.calls]
    assert names == ["allreduce_op_", "allgather_", "allgather_", "reduce_scatter_", "reduce_scatter_", "alltoall_", "alltoall_"]
    assert g.comm.calls[0][1][1] == "max"
    assert [v.numel() for v in g.comm.calls[5][1][0]] == [2, 2, 2]  # split into the group's 3 blocks
    assert world.calls == []
    with pytest.raises(ValueError, match="tensor_list has 4 tensors, world size is 3"):
        D.all_gather(lst + [torch.zeros(2)], torch.zeros(2), group=g)


def test_roots_and_peers_are_global_ranks_or_group_ranks(fabric):
    D, world = fabric(4, 2)
    g = _group(D, [0, 2, 3], 2)
    t = torch.zeros(3)
    D.broadcast(t, 3, group=g)
    D.broadcast(t, group=g, group_src=1)
    D.reduce(t, dst=0, group=g)
    D.reduce(t, group=g, group_dst=2)
    D.send(t, 3, group=g)
    D.send(t, group=g, group_dst=0)
    assert D.recv(t, 0, group=g) == 0
    assert D.recv(t, group=g, group_src=2) == 3  # returns the global rank
    D.isend(t, 0, group=g)
    D.irecv(t, group=g, group_src=0)
    got = [(c[0], c[2].get("root", c[1][1] if c[0] == "reduce_" else c[1][0][0][2] if c[0] == "p2p_" else None)) for c in g.comm.calls]
    assert got == [("broadcast_", 2), ("broadcast_", 1), ("reduce_", 0), ("reduce_", 2), ("p2p_", 2), ("p2p_", 0), ("p2p_", 0),
                   ("p2p_", 2), ("p2p_", 0), ("p2p_", 0)]
    for call in (lambda: D.broadcast(t, 1, group=g), lambda: D.reduce(t, dst=1, group=g), lambda: D.send(t, 1, group=g),
                 lambda: D.recv(t, 1, group=g), lambda: D.isend(t, 1, group=g), lambda: D.irecv(t, 1, group=g),
                 lambda: D.gather(t, None, dst=1, group=g), lambda: D.scatter(t, None, src=1, group=g),
                 lambda: D.P2POp(D.isend, t, 1, group=g)):
        with pytest.raises(ValueError, match="is not part of group"):
            call()
    with pytest.raises(ValueError, match="group_src 3 is not a rank of a group of 3"):
        D.broadcast(t, group=g, group_src=3)
    with pytest.raises(ValueError, match="Can't specify both"):
        D.broadcast(t, 0, group=g, group_src=0)
    assert world.calls == []


def test_gather_scatter_and_batches_on_a_group(fabric):
    D, _ = fabric(4, 3)
    g = _group(D, [1, 3], 3)
    t = torch.full((2,), 7.0)
    lst = [torch.zeros(2), torch.zeros(2)]
    D.gather(t, lst, dst=3, group=g)  # this rank is the root (group rank 1): one receive from group rank 0
    assert g.comm.calls[-1][1][0] == [("recv", lst[0], 0)] and torch.equal(lst[1], t)
    D.scatter(t, None, src=1, group=g)
    assert g.comm.calls[-1][1][0] == [("recv", t, 0)]
    ops = [D.P2POp(D.isend, t, 1, group=g), D.P2POp(D.irecv, t, group=g, group_peer=0)]
    assert (ops[0].peer, ops[0].group_peer, ops[1].peer, ops[1].group_peer) == (1, 0, 1, 0)
    works = D.batch_isend_irecv(ops)
    assert len(works) == 2 and g.comm.calls[-1][1][0] == [("send", t, 0), ("recv", t, 0)]
    with pytest.raises(ValueError, match="All ops need to use the same group"):
        D.batch_isend_irecv([D.P2POp(D.isend, t, 1, group=g), D.P2POp(D.isend, t, 1)])
    with pytest.raises(ValueError, match="All ops need to use the same group"):
        D.batch_isend_irecv([D.P2POp(D.isend, t, 1), D.P2POp(D.isend, t, 1, group=g)])


def test_a_non_member_does_what_torch_does(fabric):
    D, world = fabric(4, 1)
    nm = D.NON_GROUP_MEMBER
    assert nm == dist.GroupMember.NON_GROUP_MEMBER
    t = torch.zeros(3)
    warned = (lambda: D.all_reduce(t, group=nm), lambda: D.all_gather_into_tensor(t, t, group=nm),
              lambda: D.all_gather([t], t, group=nm), lambda: D.reduce_scatter_tensor(t, t, group=nm),
              lambda: D.reduce_scatter(t, [t], group=nm), lambda: D.all_to_all_single(t, t, group=nm),
              lambda: D.all_to_all([t], [t], group=nm), lambda: D.gather(t, None, group=nm), lambda: D.irecv(t, 0, group=nm),
              lambda: D.broadcast(t, group=nm, group_src=0), lambda: D.reduce(t, group=nm, group_dst=0),
              lambda: D.send(t, group=nm, group_dst=0), lambda: D.isend(t, group=nm, group_dst=0),
              lambda: D.scatter(t, None, group=nm, group_src=0), lambda: D.barrier(group=nm))
    for call in warned:
        with warnings.catch_warnings(record=True) as ws:
            warnings.simplefilter("always")
            assert call() is None
        assert [str(w.message) for w in ws][-1].endswith("on global rank 1 which does not belong to the given group.")
    with pytest.warns(UserWarning, match="does not belong"):
        assert D.recv(t, 0, group=nm) == -1
    # a global rank cannot be translated on a non-member (torch: the group is not registered)
    for call in (lambda: D.broadcast(t, 0, group=nm), lambda: D.reduce(t, 0, group=nm), lambda: D.send(t, 0, group=nm),
                 lambda: D.isend(t, 0, group=nm), lambda: D.scatter(t, None, src=0, group=nm),
                 lambda: D.P2POp(D.isend, t, 0, group=nm), lambda: D.P2POp(D.isend, t, group=nm, group_peer=0)):
        with pytest.raises(ValueError):
            call()
    assert world.calls == []


def test_any_other_group_object_is_still_refused(fabric):
    D, world = fabric(2, 0)
    t, g = torch.zeros(2), object()
    for call in (lambda: D.all_reduce(t, group=g), lambda: D.broadcast(t, 0, group=g), lambda: D.send(t, 1, group=g),
                 lambda: D.recv(t, 1, group=g), lambda: D.gather(t, None, group=g), lambda: D.barrier(group=g),
                 lambda: D.all_gather_object([None, None], 1, group=g), lambda: D.new_subgroups(1, group=g)):
        with pytest.raises(NotImplementedError, match="no subgroups"):
            call()
    from torchx_b200.nn import SyncBatchNorm

    bn = SyncBatchNorm(4, process_group=g)
    with pytest.raises(NotImplementedError, match="no subgroups"):
        bn(torch.zeros(2, 4, 3, 3))
    assert world.calls == []


class _GroupMaker(_FakeComm):
    """A world stand-in whose create_group records the lists and returns a member's communicator."""

    def create_group(self, ranks, stage_mb=0):
        self.calls.append(("create_group", (list(ranks), stage_mb), {}))
        if self.rank not in ranks:
            return None
        c = _FakeComm(len(ranks), list(ranks).index(self.rank))
        c.ranks = list(ranks)
        return c


def test_new_group_and_subgroups(monkeypatch):
    import torchx_b200.distributed as D

    world = _GroupMaker(8, 5)
    monkeypatch.setattr(D, "_COMM", world)
    g = D.new_group([6, 5, 1], stage_mb=8)
    assert isinstance(g, D.B200Group) and g.ranks == [1, 5, 6] and g.rank() == 1
    assert D.new_group([0, 2]) is D.NON_GROUP_MEMBER
    for bad in ([0, 8], [-1], [1, 1], []):
        with pytest.raises(ValueError):
            D.new_group(bad)
    cur, groups = D.new_subgroups(4)
    assert cur.ranks == [4, 5, 6, 7] and groups[0] is D.NON_GROUP_MEMBER and groups[1] is cur
    cur, groups = D.new_subgroups_by_enumeration([[0, 2, 4, 6], [1, 3, 5, 7]])
    assert cur.ranks == [1, 3, 5, 7] and cur.rank() == 2 and groups[0] is D.NON_GROUP_MEMBER
    made = [c[1] for c in world.calls if c[0] == "create_group"]
    assert made == [([1, 5, 6], 8), ([0, 2], 0), ([0, 1, 2, 3], 0), ([4, 5, 6, 7], 0), ([0, 2, 4, 6], 0), ([1, 3, 5, 7], 0)]
    with pytest.raises(ValueError, match="Rank 2 has appeared in both subgroup"):
        D.new_subgroups_by_enumeration([[0, 2], [2, 3]])
    with pytest.raises(ValueError, match="must be divisible"):
        D.new_subgroups(3)
    with pytest.raises(ValueError, match="must not exceed"):
        D.new_subgroups(16)
    with pytest.raises(ValueError, match="cannot be empty"):
        D.new_subgroups_by_enumeration([])
    assert len(world.calls) == 6  # refused before any group was made


def test_syncbatchnorm_synchronises_over_a_stand_in_group(fabric, monkeypatch):
    """A B200Group passes the layer's group check (the next check is the GPU input), and the layer's function exchanges the
    statistics on the group's communicator with counts_out of the group's size."""
    import torchx_b200.nn.batchnorm as B
    from torchx_b200.nn import SyncBatchNorm

    D, world = fabric(4, 3)
    g = _group(D, [1, 3], 3)
    bn = SyncBatchNorm.convert_sync_batchnorm(torch.nn.Sequential(torch.nn.BatchNorm2d(4)), g)[0]
    assert bn.process_group is g
    x = torch.randn(2, 4, 3, 3)
    with pytest.raises(ValueError, match="expected input tensor to be on GPU"):
        bn(x)
    monkeypatch.setattr(torch, "batch_norm_stats", lambda inp, eps: (torch.zeros(4), torch.ones(4)))
    monkeypatch.setattr(torch, "batch_norm_elemt", lambda inp, *a: inp.clone())
    B._FabricSyncBatchNorm.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, 1e-5, 0.1, g.comm)
    (name, args, kw), = g.comm.calls
    assert name == "batchnorm_stats_" and args[2] == 18.0 and kw["counts_out"].numel() == 2
    assert world.calls == []
