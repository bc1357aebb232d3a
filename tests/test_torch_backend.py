"""The "b200" torch.distributed backend without a GPU: registration, the creator's checks, the method-to-Communicator map
and the refusals, on a stand-in communicator in ``torchx_b200.distributed._COMM`` and a HashStore world."""
import pytest
import torch
import torch.distributed as dist

import torchx_b200.distributed as D
from torchx_b200.ddp.comm import Communicator
from torchx_b200.distributed import _backend as B


class _FakeStream:
    """Stands in for the communicator's ordered stream: the group's shutdown synchronises it."""

    def synchronize(self):
        pass


class _FakeComm:
    """Stands in for the native communicator: records calls; collectives write simple recognisable values."""

    def __init__(self, rank, world, accept_cpu=True):
        self.rank, self.world, self.device = rank, world, 0
        self.ordered_stream = _FakeStream()
        self.calls = []
        self.checks = 0
        self.accept_cpu = accept_cpu

    def _check_tensor(self, t):
        if not self.accept_cpu:
            Communicator._check_tensor(self, t)
        elif not t.is_contiguous():
            raise ValueError("collectives need a contiguous tensor")

    def check(self):
        self.checks += 1

    def allreduce_op_(self, t, op, stream=None):
        self.calls.append(("allreduce_op_", op, stream))
        t.add_(1)

    def broadcast_(self, t, root, stream=None):
        self.calls.append(("broadcast_", root, stream))

    def allgather_(self, out, t, stream=None):
        self.calls.append(("allgather_", tuple(out.shape), tuple(t.shape)))
        for r in range(self.world):
            out.view(self.world, -1)[r].copy_(t.reshape(-1) + 100 * r)

    def reduce_scatter_(self, out, t, op, stream=None):
        self.calls.append(("reduce_scatter_", op, t.tolist()))
        out.copy_(t.view(self.world, -1)[self.rank].view_as(out))

    def reduce_(self, t, root, op, stream=None):
        self.calls.append(("reduce_", root, op))

    def alltoall_(self, outs, ins, stream=None):
        self.calls.append(("alltoall_", [o.numel() for o in outs], [i.numel() for i in ins]))

    def p2p_(self, ops, stream=None):
        self.calls.append(("p2p_", [(k, p, t.numel()) for k, t, p in ops]))

    def barrier(self, stream=None):
        self.calls.append(("barrier",))


def _done(self, launch, tensors, outputs):
    launch("stream")
    fut = torch.futures.Future()
    fut.set_result(outputs)
    return torch._C._distributed_c10d._create_work_from_future(fut)


@pytest.fixture
def world(monkeypatch):
    """A HashStore world of 3 ranks as rank 1 sees it, on a stand-in communicator."""
    fake = _FakeComm(1, 3)
    monkeypatch.setattr(D, "_COMM", fake)
    monkeypatch.setattr(B.B200ProcessGroup, "_enqueue", _done)
    monkeypatch.setattr(B.B200ProcessGroup, "_wait_current", lambda self: None)
    monkeypatch.setattr(B.B200ProcessGroup, "barrier", lambda self, opts=None: _done(self, lambda s: self.comm.barrier(s), [], []))
    dist.init_process_group("b200", store=dist.HashStore(), rank=1, world_size=3)
    yield fake
    dist.destroy_process_group()


def test_registration_is_idempotent():
    import subprocess
    import sys

    plugin = dist.Backend._plugins["B200"]
    B.register_backend()
    assert dist.Backend._plugins["B200"] is plugin
    # a second import (a reload, in a fresh interpreter) registers again: a no-op
    code = ("import importlib, torch.distributed as dist, torchx_b200.distributed as D; p = dist.Backend._plugins['B200']; "
            "importlib.reload(D); assert dist.Backend._plugins['B200'] is p; assert dist.Backend.backend_list.count('b200') == 1")
    root = __file__.rsplit("/tests/", 1)[0]
    subprocess.run([sys.executable, "-c", code], cwd=root, check=True, timeout=300)
    assert plugin.extended_api
    assert dist.Backend.backend_capability["b200"] == ["cuda"]
    assert dist.Backend.backend_list.count("b200") == 1


def test_group_backend_and_local_device(world):
    assert dist.get_backend() == "b200"
    assert isinstance(dist.group.WORLD, B.B200ProcessGroup)
    assert dist.get_rank() == 1 and dist.get_world_size() == 3
    assert D._COMM is world and dist.group.WORLD.comm is world
    assert D.local_device() == torch.device("cuda", 0)
    assert dist.distributed_c10d._get_object_coll_device() == "cuda"


def test_full_world_new_group_shares_the_communicator(world):
    g = dist.new_group()
    assert isinstance(g, B.B200ProcessGroup) and g is not dist.group.WORLD and g.comm is world
    g2 = dist.new_group(ranks=[0, 1, 2])
    assert g2.comm is world
    t = torch.zeros(2, dtype=torch.int64)
    dist.all_reduce(t, group=g)
    assert world.calls[-1] == ("allreduce_op_", "sum", "stream")


def test_subset_group_is_refused(world):
    with pytest.raises(NotImplementedError, match="the b200 communicator has no subgroups"):
        dist.new_group(ranks=[0, 1])


class _Opts:
    def __init__(self, rank, size, ranks):
        self.group_rank, self.group_size, self.global_ranks_in_group = rank, size, ranks


def test_creator_checks_rank_and_world(monkeypatch):
    fake = _FakeComm(1, 3)
    monkeypatch.setattr(D, "_COMM", fake)
    assert B._create(_Opts(1, 3, [])).comm is fake
    assert B._create(_Opts(1, 3, [2, 0, 1])).comm is fake
    with pytest.raises(ValueError, match="rank 2 of 3 differs from the communicator's rank 1 of 3"):
        B._create(_Opts(2, 3, []))
    with pytest.raises(ValueError, match="rank 1 of 4 differs"):
        B._create(_Opts(1, 4, []))
    with pytest.raises(NotImplementedError, match="no subgroups"):
        B._create(_Opts(1, 2, [1, 2]))


def test_creator_takes_the_communicator_from_the_environment(monkeypatch):
    fake = _FakeComm(0, 2)
    monkeypatch.setattr(D, "_COMM", None)
    monkeypatch.setattr(Communicator, "from_env", classmethod(lambda cls: fake))
    assert B._create(_Opts(0, 2, [])).comm is fake
    assert D._COMM is fake


@pytest.mark.parametrize("first", ["init_pg", "init_process_group", "mini_ddp", "hook_state"])
def test_every_entry_point_shares_one_process_communicator(monkeypatch, first):
    """Whichever entry point comes first makes the communicator from the environment; the others reuse it."""
    from torchx_b200.ddp import B200HookState, DistributedDataParallel

    fake, made = _FakeComm(0, 1), []
    monkeypatch.setattr(D, "_COMM", None)
    monkeypatch.setattr(Communicator, "from_env", classmethod(lambda cls, **kw: made.append(kw) or fake))
    monkeypatch.setattr(torch.cuda, "Stream", lambda device=None: None)
    monkeypatch.setattr(torch.cuda, "Event", lambda: None)

    def mini_ddp():
        with pytest.raises(ValueError, match="parameter on cpu, communicator on cuda:0"):  # after it took the communicator
            DistributedDataParallel(torch.nn.Linear(2, 2))

    entries = {"init_pg": lambda: D.init_pg("b200"), "init_process_group": lambda: B._create(_Opts(0, 1, [])),
               "mini_ddp": mini_ddp, "hook_state": lambda: B200HookState()}
    entries.pop(first)()
    assert D._COMM is fake and made == [{}]
    for enter in entries.values():
        enter()
    assert D.init_pg("b200") == torch.device("cuda", 0) and B200HookState().comm is fake
    assert B._create(_Opts(0, 1, [])).comm is fake and made == [{}]


def test_the_group_installs_no_stream_over_an_owner():
    fake = _FakeComm(0, 2)
    owner = fake.ordered_stream
    B.B200ProcessGroup(fake)
    assert fake.ordered_stream is owner


def test_allreduce_ops_and_work(world):
    t = torch.zeros(4, dtype=torch.int32)
    for op, name in ((dist.ReduceOp.SUM, "sum"), (dist.ReduceOp.MIN, "min"), (dist.ReduceOp.MAX, "max")):
        assert dist.all_reduce(t, op=op) is None
        assert world.calls[-1] == ("allreduce_op_", name, "stream")
    f = torch.zeros(3, dtype=torch.bfloat16)
    w = dist.all_reduce(f, op=dist.ReduceOp.AVG, async_op=True)
    assert world.calls[-1] == ("allreduce_op_", "avg", "stream")
    w.wait()
    assert w.get_future().value()[0] is f and f.tolist() == [1.0, 1.0, 1.0]
    assert world.checks == 4  # the communicator's health is read before each launch


def test_gather_family(world):
    t = torch.arange(4, dtype=torch.int64)
    out = torch.empty(12, dtype=torch.int64)
    dist.all_gather_into_tensor(out, t)
    assert out.tolist() == [0, 1, 2, 3, 100, 101, 102, 103, 200, 201, 202, 203]
    lst = [torch.empty(2, 2, dtype=torch.int64) for _ in range(3)]
    dist.all_gather(lst, t.view(2, 2))
    assert [x.reshape(-1).tolist() for x in lst] == [[0, 1, 2, 3], [100, 101, 102, 103], [200, 201, 202, 203]]
    assert world.calls[-1] == ("allgather_", (3, 2, 2), (2, 2))
    with pytest.raises(ValueError, match="world size is 3"):
        dist.all_gather(lst[:2], t.view(2, 2))


def test_reduce_scatter_family(world):
    o = torch.empty(2, dtype=torch.float32)
    dist.reduce_scatter_tensor(o, torch.arange(6, dtype=torch.float32), op=dist.ReduceOp.MAX)
    assert world.calls[-1][:2] == ("reduce_scatter_", "max") and o.tolist() == [2.0, 3.0]
    dist.reduce_scatter(o, [torch.full((2,), float(r)) for r in range(3)], op=dist.ReduceOp.AVG)
    assert world.calls[-1] == ("reduce_scatter_", "avg", [0.0, 0.0, 1.0, 1.0, 2.0, 2.0]) and o.tolist() == [1.0, 1.0]
    with pytest.raises(ValueError, match="input has 5 elements, needs 3 x 2"):
        dist.reduce_scatter_tensor(o, torch.zeros(5))
    with pytest.raises(ValueError, match="every tensor of input_list must be torch.float32 with 2 elements"):
        dist.reduce_scatter(o, [torch.zeros(2), torch.zeros(3), torch.zeros(2)])


def test_broadcast_and_reduce_at_every_root(world):
    t = torch.zeros(3)
    for root in range(3):
        dist.broadcast(t, root)
        assert world.calls[-1] == ("broadcast_", root, "stream")
        dist.reduce(t, root, op=dist.ReduceOp.MIN)
        assert world.calls[-1] == ("reduce_", root, "min")


def test_all_to_all(world):
    out, inp = torch.empty(6, 2), torch.zeros(7, 2)
    dist.all_to_all_single(out, inp, output_split_sizes=[1, 0, 5], input_split_sizes=[3, 4, 0])
    assert world.calls[-1] == ("alltoall_", [2, 0, 10], [6, 8, 0])
    dist.all_to_all_single(torch.empty(6), torch.zeros(6))
    assert world.calls[-1] == ("alltoall_", [2, 2, 2], [2, 2, 2])
    with pytest.raises(ValueError, match="output_split_sizes"):
        dist.all_to_all_single(out, inp, output_split_sizes=[1, 1, 1], input_split_sizes=[3, 4, 0])
    outs, ins = [torch.empty(k) for k in (1, 2, 3)], [torch.zeros(k) for k in (3, 2, 1)]
    dist.all_to_all(outs, ins)
    assert world.calls[-1] == ("alltoall_", [1, 2, 3], [3, 2, 1])


def test_point_to_point(world):
    t = torch.zeros(5)
    dist.send(t, 2)
    assert world.calls[-1] == ("p2p_", [("send", 2, 5)])
    assert dist.recv(t, 0) == 0
    assert world.calls[-1] == ("p2p_", [("recv", 0, 5)])
    dist.isend(t, 0).wait()
    dist.irecv(t, 2).wait()
    assert world.calls[-2:] == [("p2p_", [("send", 0, 5)]), ("p2p_", [("recv", 2, 5)])]
    # torch's batch_isend_irecv calls send / recv one by one: the group launches the list as ONE batch at the first wait
    n = len(world.calls)
    reqs = dist.batch_isend_irecv([dist.P2POp(dist.isend, t, 2), dist.P2POp(dist.irecv, t, 0)])
    assert len(world.calls) == n
    reqs[1].wait()
    assert world.calls[n:] == [("p2p_", [("send", 2, 5), ("recv", 0, 5)])]
    reqs[0].wait()
    assert reqs[0].is_completed() and len(world.calls) == n + 1
    assert [x is t for x in reqs[0].get_future().value()] == [True, True]
    # pending ops launch before the group's next collective, in issue order
    w = dist.isend(t, 2)
    dist.all_reduce(torch.zeros(1))
    assert world.calls[-2:] == [("p2p_", [("send", 2, 5)]), ("allreduce_op_", "sum", "stream")]
    w.wait()
    assert world.calls[-1][0] == "allreduce_op_"
    # at most 64 ops in one launch
    works = [dist.isend(t, 0) for _ in range(65)]
    assert world.calls[-1] == ("p2p_", [("send", 0, 5)] * 64)
    works[-1].wait()
    assert world.calls[-1] == ("p2p_", [("send", 0, 5)])
    with pytest.raises(NotImplementedError, match="cannot receive from any source"):
        dist.recv(t)
    with pytest.raises(ValueError, match="can only name another rank"):
        dist.group.WORLD.send([t], 1, 0)


def test_gather_and_scatter(world):
    t = torch.ones(2)
    dist.gather(t, dst=0)  # not the root: one send
    assert world.calls[-1] == ("p2p_", [("send", 0, 2)])
    lst = [torch.zeros(2) for _ in range(3)]
    dist.gather(t, lst, dst=1)  # the root: one batch of W - 1 receives, its own tensor copied
    assert world.calls[-1] == ("p2p_", [("recv", 0, 2), ("recv", 2, 2)]) and lst[1].tolist() == [1.0, 1.0]
    dist.scatter(t, src=2)
    assert world.calls[-1] == ("p2p_", [("recv", 2, 2)])
    out = torch.zeros(2)
    dist.scatter(out, [torch.full((2,), float(r)) for r in range(3)], src=1)
    assert world.calls[-1] == ("p2p_", [("send", 0, 2), ("send", 2, 2)]) and out.tolist() == [1.0, 1.0]


def test_barrier(world):
    dist.barrier()
    assert world.calls[-1] == ("barrier",)


@pytest.mark.parametrize("dtype", [torch.float64, torch.uint8, torch.int8, torch.bool, torch.int16])
def test_reduction_dtypes_refused(world, dtype):
    t = torch.zeros(4, dtype=dtype)
    n = len(world.calls)
    with pytest.raises(TypeError, match=f"allreduce_op_: unsupported dtype {dtype}"):
        dist.all_reduce(t)
    with pytest.raises(TypeError, match=f"reduce_scatter_: unsupported dtype {dtype}"):
        dist.reduce_scatter_tensor(torch.zeros(1, dtype=dtype), torch.zeros(3, dtype=dtype))
    with pytest.raises(TypeError, match=f"reduce_: unsupported dtype {dtype}"):
        dist.reduce(t, 0)
    assert len(world.calls) == n  # refused before anything reached the communicator


def test_integer_avg_refused(world):
    with pytest.raises(TypeError, match="allreduce_op_: avg needs a floating-point tensor, got torch.int64"):
        dist.all_reduce(torch.zeros(2, dtype=torch.int64), op=dist.ReduceOp.AVG)


@pytest.mark.parametrize("op", ["PRODUCT", "BAND", "BOR", "BXOR", "PREMUL_SUM"])
def test_reduce_ops_refused(world, op):
    rop = dist._make_nccl_premul_sum(2.0) if op == "PREMUL_SUM" else getattr(dist.ReduceOp, op)
    with pytest.raises(ValueError, match="supports SUM, AVG, MIN and MAX"):
        dist.all_reduce(torch.zeros(2), op=rop)
    with pytest.raises(ValueError, match="supports SUM, AVG, MIN and MAX"):
        dist.reduce_scatter_tensor(torch.zeros(1), torch.zeros(3), op=rop)


def test_cpu_and_non_contiguous_tensors_refused(world):
    world.accept_cpu = False
    with pytest.raises(ValueError, match="tensor on cpu, communicator on cuda:0"):
        dist.all_reduce(torch.zeros(2))
    with pytest.raises(ValueError, match="tensor on cpu, communicator on cuda:0"):
        dist.broadcast(torch.zeros(2), 0)
    with pytest.raises(ValueError, match="tensor on cpu, communicator on cuda:0"):
        dist.send(torch.zeros(2), 0)
    world.accept_cpu = True
    with pytest.raises(ValueError, match="collectives need a contiguous tensor"):
        dist.all_reduce(torch.zeros(3, 4).t())


def test_refused_entry_points(world):
    g = dist.group.WORLD
    with pytest.raises(ValueError, match="only implemented for GLOO"):  # torch refuses it before reaching the group
        dist.monitored_barrier()
    with pytest.raises(NotImplementedError, match="no monitored_barrier"):
        g.monitored_barrier()
    for fn in ("allreduce_coalesced", "allgather_coalesced", "allgather_into_tensor_coalesced",
               "reduce_scatter_tensor_coalesced", "_start_coalescing", "_end_coalescing"):
        with pytest.raises(NotImplementedError, match="no coalesced collectives"):
            getattr(g, fn)()
    with pytest.raises(NotImplementedError, match="cannot receive from any source"):
        g.recv_anysource([torch.zeros(1)], 0)


def test_object_collectives_run_on_the_group(world):
    # torch's object collectives over this group: the sizes and bytes go through allgather / broadcast on the GPU device
    # (the stand-in accepts CPU tensors: the device itself is checked on the GPU)
    assert dist.distributed_c10d._get_object_coll_device(dist.group.WORLD) == "cuda"


def test_destroy_keeps_the_communicator_and_reinit_works(world):
    dist.destroy_process_group()
    assert D._COMM is world and not dist.is_initialized()
    dist.init_process_group("b200", store=dist.HashStore(), rank=1, world_size=3)
    assert dist.group.WORLD.comm is world


def test_helpers_delegate_to_the_group(world):
    t = torch.zeros(2, dtype=torch.int32)
    w = D.all_reduce(t, op=dist.ReduceOp.MAX, async_op=True)
    w.wait()
    assert world.calls[-1] == ("allreduce_op_", "max", "stream")
    D.broadcast(t, 2)
    assert world.calls[-1] == ("broadcast_", 2, "stream")
