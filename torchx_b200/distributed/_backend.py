"""The native communicator as a ``torch.distributed`` backend: ``dist.init_process_group("b200")``.

``B200ProcessGroup`` is a Python ``torch.distributed.ProcessGroup`` (torch's PythonProcessGroup path: the creator returns
the group itself, and ``dist.*``, stock ``DistributedDataParallel``, ``torch.nn.SyncBatchNorm``, torch's
``ZeroRedundancyOptimizer`` and the object collectives call its methods).  Every method is one or a few existing
``Communicator`` calls; the kernels are the fabric's sm_90a collectives.

Stream and work semantics are NCCL's (DESIGN.md 2.7):
  * every collective of the communicator is enqueued on ``comm.ordered_stream``: the group's own side stream, installed at
    creation when no mini-DDP owns the communicator, or the mini-DDP's comm stream after one is built; the stream is read
    at each call;
  * that stream first waits for the caller's current stream, and every tensor of the call is ``record_stream``-ed on it;
  * the returned work wraps a CUDA future completed on that stream: ``wait()`` makes the caller's current stream wait
    (the host does not block), ``get_future().value()`` is the list of output tensors;
  * ``send`` / ``recv`` queue their op; the queued ops launch as one ``p2p_`` batch at the first wait on one of their works,
    at the group's next collective or at 64 pending ops, so torch's ``batch_isend_irecv`` is one launch (``_P2PWork``);
  * ``barrier`` blocks the host until every rank has reached it, as NCCL's does;
  * a poisoned communicator (a kernel that gave up on a stalled peer) raises before anything is enqueued, and so does
    every call made while the current stream is being captured into a CUDA graph.
"""
from __future__ import annotations

from typing import Any, Callable, List, Sequence

import torch
import torch.distributed as dist
from torch._C._distributed_c10d import _create_work_from_future

from torchx_b200 import distributed as D
from torchx_b200.ddp._native import B2_P2P_MAX_OPS
from torchx_b200.ddp.comm import check_allgather, check_alltoall, check_peer, check_reduce_scatter, dtype_op_for

BACKEND = "b200"


class B200ProcessGroup(dist.ProcessGroup):
    """A ``torch.distributed`` process group of every rank of the native communicator ``comm``."""

    def __init__(self, comm: Any) -> None:
        super().__init__(comm.rank, comm.world)
        self.comm = comm
        self._pending: List[Any] = []  # (("send" | "recv", tensor, peer), its _P2PWork) not launched yet
        if comm.ordered_stream is None:  # no mini-DDP owns the communicator: this group's collectives get a stream of their own
            comm.ordered_stream = torch.cuda.Stream(device=comm.device)

    def getBackendName(self) -> str:  # noqa: N802 (torch's name)
        return BACKEND

    @property
    def _device_types(self) -> List[torch.device]:
        """The object collectives and ``barrier`` pick their device from this: the communicator's GPU, not the host."""
        return [torch.device("cuda")]

    # ---- launch ---------------------------------------------------------------------------------------------------------
    def _guard(self, flush: bool = True) -> None:
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("the b200 process group cannot be captured into a CUDA graph: its collectives run on the "
                               "communicator's stream, outside the capture; capture the Communicator calls instead")
        self.comm.check()
        if flush:  # send / recv ops issued before this collective launch first
            self._flush()

    def _check(self, tensors: Sequence[torch.Tensor]) -> None:
        for t in tensors:
            self.comm._check_tensor(t)

    def _wait_current(self) -> None:
        """The ordered stream waits for the work issued so far on the caller's current stream."""
        self.comm.ordered_stream.wait_stream(torch.cuda.current_stream(self.comm.device))

    def _enqueue(self, launch: Callable[[Any], None], tensors: Sequence[torch.Tensor],
                 outputs: List[torch.Tensor]) -> Any:
        """Run ``launch(stream)`` on the communicator's ordered stream after the caller's current stream; return the work."""
        comm = self.comm
        dev = torch.device("cuda", comm.device)
        s = comm.ordered_stream
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            launch(s)
            for t in tensors:
                t.record_stream(s)
            fut = torch.futures.Future(devices=[dev])
            fut.set_result(outputs)
        return _create_work_from_future(fut)

    def _op(self, op: Any, dtype: torch.dtype, fn: str) -> str:
        name = D.reduce_op_name(op)
        dtype_op_for(dtype, name, fn)
        return name

    def _root(self, fn: str, name: str, opts: Any) -> int:
        return D._resolve(fn, None, name=name, r=opts.rootRank, world=self.comm)[1]

    @staticmethod
    def _one(tensors: Sequence[torch.Tensor], fn: str) -> torch.Tensor:
        if len(tensors) != 1:
            raise ValueError(f"{fn}: the b200 process group takes one tensor per call, got {len(tensors)}")
        return tensors[0]

    # ---- collectives ----------------------------------------------------------------------------------------------------
    def allreduce(self, tensors: List[torch.Tensor], opts: Any) -> Any:
        self._guard()
        t = self._one(tensors, "allreduce")
        name = self._op(opts.reduceOp, t.dtype, "allreduce_op_")
        self._check([t])
        return self._enqueue(lambda s: self.comm.allreduce_op_(t, name, stream=s), [t], [t])

    def broadcast(self, tensors: List[torch.Tensor], opts: Any) -> Any:
        self._guard()
        t = self._one(tensors, "broadcast")
        root = self._root("broadcast", "src", opts)
        self._check([t])
        return self._enqueue(lambda s: self.comm.broadcast_(t, root=root, stream=s), [t], [t])

    def _allgather_base(self, output: torch.Tensor, input: torch.Tensor, opts: Any = None) -> Any:  # noqa: A002
        self._guard()
        check_allgather(self.comm, output, input)
        return self._enqueue(lambda s: self.comm.allgather_(output, input, stream=s), [output, input], [output])

    def allgather(self, output_tensors: List[List[torch.Tensor]], input_tensors: List[torch.Tensor], opts: Any = None) -> Any:
        self._guard()
        t = self._one(input_tensors, "allgather")
        outs = self._one(output_tensors, "allgather")
        launch = D._all_gather(self.comm, outs, t)
        self._check([t, *outs])
        return self._enqueue(launch, [t, *outs], list(outs))

    def _reduce_scatter_base(self, output: torch.Tensor, input: torch.Tensor, opts: Any) -> Any:  # noqa: A002
        self._guard()
        name = D.reduce_op_name(opts.reduceOp)
        check_reduce_scatter(self.comm, output, input, name)
        return self._enqueue(lambda s: self.comm.reduce_scatter_(output, input, name, stream=s), [output, input], [output])

    def reduce_scatter(self, output_tensors: List[torch.Tensor], input_tensors: List[List[torch.Tensor]], opts: Any) -> Any:
        self._guard()
        out = self._one(output_tensors, "reduce_scatter")
        ins = self._one(input_tensors, "reduce_scatter")
        launch = D._reduce_scatter(self.comm, out, ins, self._op(opts.reduceOp, out.dtype, "reduce_scatter_"))
        self._check([out, *ins])
        return self._enqueue(launch, [out, *ins], [out])

    def reduce(self, tensors: List[torch.Tensor], opts: Any) -> Any:
        self._guard()
        t = self._one(tensors, "reduce")
        name = self._op(opts.reduceOp, t.dtype, "reduce_")
        root = self._root("reduce", "dst", opts)
        self._check([t])
        return self._enqueue(lambda s: self.comm.reduce_(t, root, name, stream=s), [t], [t])

    def alltoall_base(self, output: torch.Tensor, input: torch.Tensor, output_split_sizes: List[int],  # noqa: A002
                      input_split_sizes: List[int], opts: Any = None) -> Any:
        self._guard()
        self._check([output, input])
        launch = D._all_to_all_single(self.comm, output, input, output_split_sizes, input_split_sizes)
        return self._enqueue(launch, [output, input], [output])

    def alltoall(self, output_tensors: List[torch.Tensor], input_tensors: List[torch.Tensor], opts: Any = None) -> Any:
        self._guard()
        check_alltoall(self.comm.world, output_tensors, input_tensors)
        self._check([*output_tensors, *input_tensors])
        outs, ins = list(output_tensors), list(input_tensors)
        return self._enqueue(lambda s: self.comm.alltoall_(outs, ins, stream=s), [*outs, *ins], outs)

    # ---- point to point -------------------------------------------------------------------------------------------------
    def _p2p(self, kind: str, tensors: List[torch.Tensor], peer: int) -> Any:
        """Queue one send / recv in the pending batch (see ``_P2PWork``); the ordered stream waits for the current one now,
        so the batch reads and writes the tensor after the work issued before this call."""
        self._guard(flush=False)
        t = self._one(tensors, kind)
        p = check_peer(0, peer, self.comm.rank, self.comm.world)
        self._check([t])
        if len(self._pending) == B2_P2P_MAX_OPS:
            self._flush()
        self._wait_current()
        work = _P2PWork(self)
        self._pending.append(((kind, t, p), work))
        return work

    def _flush(self) -> None:
        """Launch the pending send / recv ops as one ``p2p_`` batch, in issue order."""
        if not self._pending:
            return
        pending, self._pending = self._pending, []
        ops = [op for op, _ in pending]
        tensors = [t for _, t, _ in ops]
        work = self._enqueue(lambda s: self.comm.p2p_(ops, stream=s), tensors, tensors)
        for _, w in pending:
            w._work = work

    def send(self, tensors: List[torch.Tensor], dstRank: int, tag: int = 0) -> Any:  # noqa: N803 (torch's names)
        return self._p2p("send", tensors, dstRank)

    def recv(self, tensors: List[torch.Tensor], srcRank: int, tag: int = 0) -> Any:  # noqa: N803
        return self._p2p("recv", tensors, srcRank)

    def recv_anysource(self, tensors: List[torch.Tensor], tag: int = 0) -> Any:
        raise NotImplementedError(D._NO_ANY_SOURCE)

    def gather(self, output_tensors: List[List[torch.Tensor]], input_tensors: List[torch.Tensor], opts: Any) -> Any:
        """``D.gather``'s batches: the root receives W - 1 messages in one launch and copies its own tensor."""
        self._guard()
        t = self._one(input_tensors, "gather")
        dst = self._root("gather", "dst", opts)
        gl = self._one(output_tensors, "gather") if output_tensors and any(output_tensors) else []
        launch = D._gather(self.comm, t, gl, dst)
        self._check([t, *gl])
        return self._enqueue(launch, [t, *gl], list(gl))

    def scatter(self, output_tensors: List[torch.Tensor], input_tensors: List[List[torch.Tensor]], opts: Any) -> Any:
        """``D.scatter``'s batches: the root sends W - 1 messages in one launch and copies its own block."""
        self._guard()
        t = self._one(output_tensors, "scatter")
        src = self._root("scatter", "src", opts)
        sl = self._one(input_tensors, "scatter") if input_tensors and any(input_tensors) else []
        launch = D._scatter(self.comm, t, sl, src)
        self._check([t, *sl])
        return self._enqueue(launch, [t, *sl], [t])

    def barrier(self, opts: Any = None) -> Any:
        """Every rank has reached the barrier when it returns: the kernel runs on the ordered stream and the host waits for
        it, as NCCL's barrier does."""
        self._guard()
        work = self._enqueue(lambda s: self.comm.barrier(stream=s), [], [])
        self.comm.ordered_stream.synchronize()
        self.comm.check()
        return work

    # ---- refused --------------------------------------------------------------------------------------------------------
    def monitored_barrier(self, *args: Any, **kwargs: Any) -> Any:
        raise NotImplementedError("the b200 process group has no monitored_barrier: use barrier")

    def _no_coalescing(self, *args: Any, **kwargs: Any) -> Any:
        raise NotImplementedError("the b200 process group has no coalesced collectives: issue them one by one")

    allreduce_coalesced = allgather_coalesced = allgather_into_tensor_coalesced = _no_coalescing
    reduce_scatter_tensor_coalesced = _start_coalescing = _end_coalescing = _no_coalescing

    def shutdown(self) -> None:
        """``destroy_process_group``: the group's pending collectives finish; the communicator stays (``_COMM``)."""
        self._flush()
        s = self.comm.ordered_stream
        if s is not None and torch.cuda.is_available():
            s.synchronize()


class _P2PWork(dist.Work):
    """The work of one send / recv.  The op waits in its group's pending batch until a work of the batch is waited, polled
    or asked for its future, the group runs another collective, or 64 ops are pending; then the whole batch is ONE
    ``p2p_`` launch.  So torch's ``batch_isend_irecv`` - which calls a Python group's ``send`` / ``recv`` one by one - gets
    one launch for its list, as NCCL's grouped batch does, and a ring of messages past ``p2p_eager_bytes`` makes progress
    whatever the order of its ops.  ``get_future().value()`` is the batch's tensors."""

    def __init__(self, group: "B200ProcessGroup") -> None:
        super().__init__()
        self._group = group
        self._work: Any = None

    def _launched(self) -> Any:
        if self._work is None:
            self._group._flush()
        return self._work

    def wait(self, timeout: Any = None) -> bool:
        self._launched().wait()
        return True

    def is_completed(self) -> bool:
        return self._launched().is_completed()

    def get_future(self) -> Any:
        return self._launched().get_future()


def _create(opts: Any, pg_options: Any = None) -> B200ProcessGroup:
    """The creator ``init_process_group`` / ``new_group`` call: one group on the process communicator (``_COMM``, made from
    the environment if ``init_pg("b200")`` did not make it).  The store is not used."""
    ranks = list(opts.global_ranks_in_group)
    comm = D.process_communicator()
    if ranks and sorted(ranks) != list(range(comm.world)):
        raise NotImplementedError("the b200 communicator has no subgroups: a b200 group must hold every rank")
    if opts.group_rank != comm.rank or opts.group_size != comm.world:
        raise ValueError(f"b200 process group: rank {opts.group_rank} of {opts.group_size} differs from the communicator's "
                         f"rank {comm.rank} of {comm.world}")
    return B200ProcessGroup(comm)


def register_backend() -> None:
    """Register ``"b200"`` with ``torch.distributed`` for CUDA; a second call is a no-op."""
    if BACKEND.upper() in dist.Backend._plugins:
        return
    dist.Backend.register_backend(BACKEND, _create, extended_api=True, devices=["cuda"])
