"""reduce to a root and the object collectives without a GPU: the header entry and binding of b2_reduce, its checks in
b2_allreduce_op's order, Communicator.reduce_'s argument checks, and torchx_b200.distributed's reduce and six object
collectives on a stand-in communicator (which fabric calls, with what sizes; the pickle round trip; the argument errors)
and under real 2- and 3-rank gloo process groups, where they are torch.distributed's own.  The GPU side:
tests/test_reduce_gpu.py and tests/test_object_collectives_gpu.py."""
import ctypes
import os
import re

import pytest
import torch
import torch.distributed as dist

from tests.test_p2p import _bare_communicator
from torchx_b200.ddp import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_reduce_and_the_binding_matches():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    decl = re.search(r"int\s+b2_reduce\(([^)]*)\);", src)
    assert decl, "b2_reduce is not declared"
    params = [" ".join(p.split()) for p in decl.group(1).split(",")]
    assert params == ["b2_comm_t* comm", "void* buf", "size_t n_elems", "int dtype", "int op", "int root", "void* stream"]
    assert re.search(r"\*\s+b2_reduce\s+<- `dist\.reduce`", src)
    version = re.search(r"#define B2_ABI_VERSION \d+ /\*(.*?)\*/", src, re.S).group(1)
    assert re.search(r"\bb2_reduce\b", version)
    L = N.lib()
    assert "b2_reduce" in N.SYMBOLS
    assert L.b2_reduce.restype is ctypes.c_int
    assert L.b2_reduce.argtypes == [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_void_p]


def test_argument_validation_without_a_gpu():
    """dtype and op first (even when n_elems == 0), then n_elems == 0 is a no-op, then a null communicator."""
    L = N.lib()
    buf = ctypes.c_void_p(4096)
    assert L.b2_reduce(None, buf, 8, 9, N.B2_OP_SUM, 0, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"b2_reduce: unknown dtype 9"
    assert L.b2_reduce(None, buf, 0, N.B2_DT_FLOAT32, 7, 0, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"b2_reduce: unknown op 7"
    for dt, name in ((N.B2_DT_INT32, b"int32"), (N.B2_DT_INT64, b"int64")):
        for n in (0, 8):
            assert L.b2_reduce(None, buf, n, dt, N.B2_OP_AVG, 0, None) == N.B2_EINVAL
            assert L.b2_last_error() == b"b2_reduce: AVG needs a floating-point dtype, got " + name
    for dt in (N.B2_DT_INT32, N.B2_DT_INT64, N.B2_DT_FLOAT32, N.B2_DT_BFLOAT16, N.B2_DT_FLOAT16):
        for op in (N.B2_OP_SUM, N.B2_OP_MIN, N.B2_OP_MAX):
            assert L.b2_reduce(None, None, 0, dt, op, -5, None) == N.B2_OK  # nothing else is read
            assert L.b2_reduce(None, buf, 8, dt, op, 0, None) == N.B2_EINVAL
            assert L.b2_last_error() == b"null communicator"
    assert L.b2_reduce(None, None, 8, N.B2_DT_BFLOAT16, N.B2_OP_AVG, 99, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"null communicator"


def test_communicator_reduce_checks_dtype_op_root_and_tensor():
    c = _bare_communicator(3, rank=1)
    t = torch.zeros(4)
    with pytest.raises(TypeError, match="reduce_: unsupported dtype torch.uint8"):
        c.reduce_(torch.zeros(4, dtype=torch.uint8), 0)
    with pytest.raises(TypeError, match="reduce_: avg needs a floating-point tensor, got torch.int64"):
        c.reduce_(torch.zeros(4, dtype=torch.int64), 0, "avg")
    with pytest.raises(ValueError, match="reduce_: unsupported op 'prod'"):
        c.reduce_(t, 0, "prod")
    for root in (3, -1, True, None, 1.0, "0"):
        with pytest.raises(ValueError, match=f"reduce_: root {re.escape(repr(root))} is not a rank of a world of 3"):
            c.reduce_(t, root)
    with pytest.raises(ValueError, match="tensor on cpu, communicator on cuda:0"):
        c.reduce_(t, 2)
    with pytest.raises(ValueError, match="tensor on cpu, communicator on cuda:0"):
        c.reduce_(torch.zeros(4, 4).t(), 0)


# ---- torchx_b200.distributed on a stand-in communicator --------------------------------------------------------------
class _LoopComm:
    """Stands in for the native communicator.  Records every call as (name, dtype, shape[, root or peer]).  What a rank
    sends (a send, or a broadcast from this rank) is queued, and what it receives (a recv, or a broadcast from another
    rank) is taken from that queue, so one stand-in plays both ends of an exchange.  allgather_ gives every rank's block
    this rank's input."""

    def __init__(self, world, rank=0):
        self.world, self.rank, self.device = world, rank, 0
        self.calls, self.queue = [], []

    def reduce_(self, t, root, op="sum", stream=None):
        self.calls.append(("reduce", t.dtype, tuple(t.shape), root, op))

    def allgather_(self, out, t, stream=None):
        self.calls.append(("allgather", t.dtype, tuple(out.shape)))
        out.view(self.world, -1).copy_(t.reshape(1, -1))

    def broadcast_(self, t, root=0, stream=None):
        self.calls.append(("broadcast", t.dtype, tuple(t.shape), root))
        if root == self.rank:
            self.queue.append(t.clone())
        else:
            t.copy_(self.queue.pop(0))

    def p2p_(self, ops, stream=None):
        self.calls.append([(kind, t.dtype, tuple(t.shape), peer) for kind, t, peer in ops])
        for kind, t, _ in ops:
            if kind == "send":
                self.queue.append(t.clone())
            else:
                t.copy_(self.queue.pop(0))

    @property
    def p2p_eager_bytes(self):
        return 8 * (512 << 10) - 128


@pytest.fixture
def fabric(monkeypatch):
    """A stand-in communicator of `world` ranks with this rank `rank`; the object collectives build their tensors on the
    CPU instead of the communicator's device."""
    import torchx_b200.distributed as D

    assert not dist.is_initialized()
    monkeypatch.setattr(D, "_comm_device", lambda: torch.device("cpu"))

    def make(world, rank=0):
        fake = _LoopComm(world, rank)
        monkeypatch.setattr(D, "_COMM", fake)
        return D, fake

    return make


OBJECTS = [None, [], {"a": {"t": torch.arange(3, dtype=torch.int16), "s": "x"}, "b": [1, (2.5, None)]},
           bytes(range(256)) * ((5 << 20) // 256)]  # the last one larger than p2p_eager_bytes


def _same(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a, b)
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def _nbytes(obj):
    import pickle

    return len(pickle.dumps(obj))


def test_reduce_is_one_fabric_call(fabric):
    D, fake = fabric(3, rank=2)
    t = torch.zeros(5, dtype=torch.int64)
    assert D.reduce(t, 1) is None
    assert D.reduce(t, dst=0, op=dist.ReduceOp.MIN, group=dist.group.WORLD) is None
    assert fake.calls == [("reduce", torch.int64, (5,), 1, "sum"), ("reduce", torch.int64, (5,), 0, "min")]
    for dst in (3, -1, True, None):
        with pytest.raises(ValueError, match=f"reduce: dst {re.escape(repr(dst))} is not a rank of a world of 3"):
            D.reduce(t, dst)
    with pytest.raises(ValueError, match="supports SUM, AVG, MIN and MAX"):
        D.reduce(t, 0, op=dist.ReduceOp.PRODUCT)
    with pytest.raises(NotImplementedError, match="no subgroups"):
        D.reduce(t, 0, group=object())
    with pytest.raises(NotImplementedError, match="no work handles"):
        D.reduce(t, 0, async_op=True)
    assert len(fake.calls) == 2


@pytest.mark.parametrize("obj", OBJECTS, ids=["none", "empty", "nested", "big"])
def test_all_gather_object_two_allgathers(fabric, obj):
    D, fake = fabric(3, rank=1)
    out = [0, 0, 0]
    assert D.all_gather_object(out, obj) is None
    n = _nbytes(obj)
    assert fake.calls == [("allgather", torch.int64, (3,)), ("allgather", torch.uint8, (3 * n,))]
    assert all(_same(o, obj) for o in out)


@pytest.mark.parametrize("obj", OBJECTS, ids=["none", "empty", "nested", "big"])
def test_send_recv_object_list_round_trip(fabric, obj):
    D, fake = fabric(2, rank=0)
    objs = [obj, "tail", 7]
    sizes = [_nbytes(o) for o in objs]
    assert D.send_object_list(objs, dst=1, use_batch=True) is None
    assert fake.calls == [[("send", torch.int64, (3,), 1)], [("send", torch.uint8, (sum(sizes),), 1)]]
    got = [None] * 3
    assert D.recv_object_list(got, src=1, group_src=1) == 1  # the stand-in hands this rank what it just sent
    assert fake.calls[2:] == [[("recv", torch.int64, (3,), 1)], [("recv", torch.uint8, (sum(sizes),), 1)]]
    assert _same(got, objs)


@pytest.mark.parametrize("obj", OBJECTS, ids=["none", "empty", "nested", "big"])
def test_broadcast_object_list_root_then_peer(fabric, obj):
    D, fake = fabric(4, rank=2)
    objs = [obj, {"k": 1}]
    before = list(objs)
    n = sum(_nbytes(o) for o in objs)
    assert D.broadcast_object_list(objs, src=2) is None
    assert objs == before or _same(objs, before)  # the source's list is left as it is
    fake.rank = 0
    got = [None, None]
    D.broadcast_object_list(got, group_src=2)
    assert fake.calls == [("broadcast", torch.int64, (2,), 2), ("broadcast", torch.uint8, (n,), 2)] * 2
    assert _same(got, objs)


def test_gather_object_sizes_then_padded_gather(fabric):
    D, fake = fabric(3, rank=0)
    obj = OBJECTS[2]
    n = _nbytes(obj)
    D.gather_object(obj, None, dst=2)  # a non-destination rank: one send of the padded bytes
    assert fake.calls == [("allgather", torch.int64, (3,)), [("send", torch.uint8, (n,), 2)]]
    fake.calls, fake.queue = [], [fake.queue[0]] * 2  # the destination receives rank 0's and rank 1's blocks
    fake.rank = 2
    out = [None] * 3
    D.gather_object(obj, out, dst=2, group_dst=2)
    assert fake.calls == [("allgather", torch.int64, (3,)), [("recv", torch.uint8, (n,), 0), ("recv", torch.uint8, (n,), 1)]]
    assert all(_same(o, obj) for o in out)


def test_scatter_object_list_sizes_then_padded_scatter(fabric):
    D, fake = fabric(3, rank=1)
    ins = [OBJECTS[3], None, {"r": 2}]
    sizes = [_nbytes(o) for o in ins]
    out = [None]
    D.scatter_object_list(out, ins, src=1)
    assert out[0] is None
    assert fake.calls == [("broadcast", torch.int64, (3,), 1),
                          [("send", torch.uint8, (max(sizes),), 0), ("send", torch.uint8, (max(sizes),), 2)]]
    fake.calls, fake.rank = [], 2  # rank 2: the sizes, then its padded block
    fake.queue = [fake.queue[0], fake.queue[2]]
    D.scatter_object_list(out, None, src=1)
    assert fake.calls == [("broadcast", torch.int64, (3,), 1), [("recv", torch.uint8, (max(sizes),), 1)]]
    assert out == [{"r": 2}]


def test_object_collectives_check_their_arguments(fabric):
    D, fake = fabric(2, rank=0)
    with pytest.raises(ValueError, match=r"Argument ``gather_list`` must be specified on destination rank\."):
        D.gather_object(1, None, dst=0)
    with pytest.raises(ValueError, match=r"Argument ``gather_list`` must NOT be specified on non-destination ranks\."):
        D.gather_object(1, [None, None], dst=1)
    with pytest.raises(ValueError, match="Expected argument scatter_object_output_list to be a list of size at least 1."):
        D.scatter_object_list([], [1, 2])
    with pytest.raises(ValueError, match="source rank must provide non-None scatter_object_input_list"):
        D.scatter_object_list([None], None, src=0)
    with pytest.raises(ValueError, match="scatter_object_input_list has 3 objects, world size is 2"):
        D.scatter_object_list([None], [1, 2, 3], src=0)
    with pytest.raises(ValueError, match="group_src 1 differs from src 0"):
        D.broadcast_object_list([1], src=0, group_src=1)
    with pytest.raises(ValueError, match="group_dst 0 differs from dst 1"):
        D.send_object_list([1], dst=1, group_dst=0)
    with pytest.raises(ValueError, match="send_object_list: dst must be given"):
        D.send_object_list([1])
    with pytest.raises(NotImplementedError, match="cannot receive from any source"):
        D.recv_object_list([None])
    with pytest.raises(ValueError, match="recv_object_list: src 2 is not a rank of a world of 2"):
        D.recv_object_list([None], src=2)
    with pytest.raises(ValueError, match="broadcast_object_list: device cuda:1 is not the b200 communicator's device cpu"):
        D.broadcast_object_list([1], device="cuda:1")
    with pytest.raises(ValueError, match="send_object_list: device meta is not the b200 communicator's device cpu"):
        D.send_object_list([1], dst=1, device="meta")
    for call in (lambda g: D.all_gather_object([None, None], 1, group=g), lambda g: D.gather_object(1, [0, 0], group=g),
                 lambda g: D.broadcast_object_list([1], group=g), lambda g: D.scatter_object_list([None], [1, 2], group=g),
                 lambda g: D.send_object_list([1], 1, group=g), lambda g: D.recv_object_list([None], 1, group=g)):
        with pytest.raises(NotImplementedError, match="no subgroups"):
            call(object())
    assert fake.calls == []


def test_helpers_delegate_without_the_native_communicator(monkeypatch):
    import torchx_b200.distributed as D

    monkeypatch.setattr(D, "_COMM", None)
    names = ("reduce", "all_gather_object", "gather_object", "broadcast_object_list", "scatter_object_list",
             "send_object_list", "recv_object_list")
    seen = []
    for name in names:
        monkeypatch.setattr(dist, name, lambda *a, _n=name, **k: seen.append((_n, a, k)) or _n)
    t = torch.zeros(2)
    assert D.reduce(t, 1, async_op=True) == "reduce"
    assert D.all_gather_object([None], 5) == "all_gather_object"
    assert D.gather_object(5, None, dst=1, group_dst=1) == "gather_object"
    assert D.broadcast_object_list([1], src=1, device="cpu") == "broadcast_object_list"
    assert D.scatter_object_list([None], None, src=1) == "scatter_object_list"
    assert D.send_object_list([1], dst=1, use_batch=True) == "send_object_list"
    assert D.recv_object_list([None], src=0) == "recv_object_list"
    assert [s[0] for s in seen] == list(names)
    assert seen[0][2] == {"op": dist.ReduceOp.SUM, "group": None, "async_op": True}
    assert seen[5][2]["use_batch"] is True and seen[2][2]["group_dst"] == 1


# ---- under real gloo process groups (CPU): every helper is torch.distributed's own ----------------------------------
def _gloo_rank(rank, world, store, out):
    import pickle

    import torchx_b200.distributed as D

    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        res = {}
        root = world - 1
        for name, mod in (("ours", D), ("torch", dist)):
            t = torch.tensor([rank + 1, -rank, 1 << 40], dtype=torch.int64)
            mod.reduce(t, root, op=dist.ReduceOp.MAX)
            f = torch.tensor([0.5 * rank, 1.0])
            mod.reduce(f, dst=0)
            ag = [None] * world
            mod.all_gather_object(ag, {"rank": rank, "t": torch.arange(rank + 1)})
            gl = [None] * world if rank == root else None
            mod.gather_object([rank] * rank, gl, dst=root)
            bl = ["dir", 3, {"seed": 1}] if rank == 0 else [None] * 3
            mod.broadcast_object_list(bl, src=0)
            so = [None]
            mod.scatter_object_list(so, [f"to {q}" for q in range(world)] if rank == root else None, src=root)
            if rank == 0:
                mod.send_object_list([{"x": 1}, None], dst=1)
                src = None
                back = None
            elif rank == 1:
                back = [None, None]
                src = mod.recv_object_list(back, src=0)
            else:
                src = back = None
            res[name] = pickle.dumps((t, f, ag, gl, bl, so, back, src))
        with open(out, "wb") as fh:
            pickle.dump(res, fh)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_helpers_are_torch_distributed_under_a_real_gloo_group(tmp_path, world):
    import multiprocessing as mp
    import pickle

    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_gloo_rank, args=(r, world, str(tmp_path / "store"), str(tmp_path / f"r{r}.pkl")))
             for r in range(world)]
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
    assert [p.exitcode for p in procs] == [0] * world
    for r in range(world):
        res = pickle.load(open(tmp_path / f"r{r}.pkl", "rb"))
        ours, theirs = pickle.loads(res["ours"]), pickle.loads(res["torch"])
        assert _same(ours, theirs), (r, ours, theirs)
        t, f, ag, gl, bl, so, back, src = ours
        if r == world - 1:
            assert t.tolist() == [world, 0, 1 << 40] and gl == [[q] * q for q in range(world)]
        assert so == [f"to {r}"] and bl == ["dir", 3, {"seed": 1}] and [a["rank"] for a in ag] == list(range(world))
        if r == 1:
            assert back == [{"x": 1}, None] and src == 0
