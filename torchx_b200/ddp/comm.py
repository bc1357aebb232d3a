"""Communicator: the worker-side handle on the NVSwitch peer-buffer fabric.

Replaces, for workers launched by the ``local_cuda`` scheduler, what ``torchx.distributed.init_pg`` obtains
from ``torch.distributed.init_process_group("nccl")`` (reference torchx/distributed/__init__.py:164-225):
rank/world discovery from the torchrun env contract, device pinning, and the collectives the DDP path needs.
torch is used for tensors and streams only.
"""
from __future__ import annotations

import ctypes
import operator
import os
from typing import List, Optional, Sequence

import torch

from . import _native as N

_MODE_FOR = {
    ("f32", "bf16"): N.B2_F32_WIRE_BF16,
    ("f32", "f32"): N.B2_F32,
    ("f32", "f16"): N.B2_F32_WIRE_F16,
    ("bf16", "bf16"): N.B2_BF16,
    ("f16", "f16"): N.B2_F16,
}
# b2_allreduce_op: the dtypes and ops it takes (include/b200ddp.h)
EXACT_DTYPES = {torch.int32: N.B2_DT_INT32, torch.int64: N.B2_DT_INT64, torch.float32: N.B2_DT_FLOAT32,
                torch.bfloat16: N.B2_DT_BFLOAT16, torch.float16: N.B2_DT_FLOAT16}
REDUCE_OPS = {"sum": N.B2_OP_SUM, "avg": N.B2_OP_AVG, "min": N.B2_OP_MIN, "max": N.B2_OP_MAX}
ALGOS = {"auto": N.B2_ALGO_AUTO, "oneshot": N.B2_ALGO_ONESHOT, "twoshot": N.B2_ALGO_TWOSHOT, "twoshot_pipe": N.B2_ALGO_TWOSHOT_PIPE,
         "nvls": N.B2_ALGO_NVLS, "twoshot_ll": N.B2_ALGO_TWOSHOT_LL}


def mode_for(tensor: torch.Tensor, wire: str = "bf16") -> int:
    """The B2_* mode for a bucket of this dtype: fp32 buckets take the wire format `wire` ("bf16", "f16" or "f32"); a
    16-bit bucket is its own wire format whatever `wire` says."""
    if tensor.dtype == torch.float32:
        key = ("f32", wire)
    elif tensor.dtype == torch.bfloat16:
        key = ("bf16", "bf16")
    elif tensor.dtype == torch.float16:
        key = ("f16", "f16")
    else:
        raise TypeError(f"unsupported gradient dtype {tensor.dtype}; expected float32, bfloat16 or float16")
    if key not in _MODE_FOR:
        raise ValueError(f"unsupported wire format {wire!r} for dtype {tensor.dtype}")
    return _MODE_FOR[key]


def dtype_op_for(dtype: torch.dtype, op: str, fn: str = "allreduce_op_"):
    """(B2_DT_*, B2_OP_*) of an allreduce_op_ or reduce_scatter_ call.  TypeError for a dtype it does not take and for
    "avg" on an integer dtype, ValueError for an op it does not know."""
    if dtype not in EXACT_DTYPES:
        raise TypeError(f"{fn}: unsupported dtype {dtype}; expected int32, int64, float32, bfloat16 or float16")
    if op not in REDUCE_OPS:
        raise ValueError(f"{fn}: unsupported op {op!r}; expected one of {sorted(REDUCE_OPS)}")
    if op == "avg" and not dtype.is_floating_point:
        raise TypeError(f"{fn}: avg needs a floating-point tensor, got {dtype}")
    return EXACT_DTYPES[dtype], REDUCE_OPS[op]


def as_rank(x) -> Optional[int]:
    """``x`` as a rank number if it is an integer as torch takes one (a Python or numpy integer, not a bool), else None."""
    if isinstance(x, bool):
        return None
    try:
        return operator.index(x)
    except TypeError:
        return None


# ---- checks shared with the "b200" process group, which makes them before it enqueues anything -----------------------
def check_allgather(comm, out: torch.Tensor, t: torch.Tensor) -> None:
    """``allgather_``'s checks: ``out`` has ``t``'s dtype and world x its size, both tensors on ``comm``'s device."""
    if out.dtype != t.dtype:
        raise TypeError(f"allgather_: out is {out.dtype}, input is {t.dtype}")
    comm._check_tensor(out)
    comm._check_tensor(t)
    if out.numel() != comm.world * t.numel():
        raise ValueError(f"allgather_: out has {out.numel()} elements, needs {comm.world} x {t.numel()}")


def check_reduce_scatter(comm, out: torch.Tensor, t: torch.Tensor, op: str):
    """``reduce_scatter_``'s checks: the dtype and op, ``t`` of ``out``'s dtype and world x its size, both tensors on
    ``comm``'s device.  Returns (B2_DT_*, B2_OP_*)."""
    dt, code = dtype_op_for(t.dtype, op, "reduce_scatter_")
    if out.dtype != t.dtype:
        raise TypeError(f"reduce_scatter_: out is {out.dtype}, input is {t.dtype}")
    if t.numel() != comm.world * out.numel():
        raise ValueError(f"reduce_scatter_: input has {t.numel()} elements, needs {comm.world} x {out.numel()}")
    comm._check_tensor(out)
    comm._check_tensor(t)
    return dt, code


def check_alltoall(world: int, outs: Sequence[torch.Tensor], ins: Sequence[torch.Tensor]) -> None:
    """``alltoall_``'s list checks: world tensors each way, all of one dtype."""
    if len(outs) != world or len(ins) != world:
        raise ValueError(f"alltoall_: needs {world} output and {world} input tensors, got {len(outs)} and {len(ins)}")
    dtypes = {t.dtype for t in (*outs, *ins)}
    if len(dtypes) > 1:
        raise TypeError(f"alltoall_: every tensor must have one dtype, got {sorted(str(d) for d in dtypes)}")


def check_peer(k: int, peer, rank: int, world: int) -> int:
    """The peer of op ``k`` of a ``p2p_`` batch as an int: another rank of the world."""
    p = as_rank(peer)
    if p is None or not 0 <= p < world or p == rank:
        raise ValueError(f"p2p_: op {k} names peer {peer!r}; rank {rank} of {world} can only name another rank")
    return p


def _stream_arg(stream: Optional[torch.cuda.Stream], device: int) -> ctypes.c_void_p:
    """The cudaStream_t argument of a library call: ``stream``, or the device's current stream."""
    s = stream if stream is not None else torch.cuda.current_stream(device)
    return ctypes.c_void_p(s.cuda_stream)


def default_shm_name() -> str:
    """Name of the rendezvous control block.  The ``local_cuda`` scheduler exports B2_SHM_NAME; under a plain
    ``torchrun`` (the bench driver) all workers share a parent agent and a MASTER_PORT, which is unique per job
    on one box."""
    name = os.environ.get("B2_SHM_NAME")
    if name:
        return name
    run_id = os.environ.get("TORCHELASTIC_RUN_ID", "none")
    port = os.environ.get("MASTER_PORT", "0")
    return f"/b2_{os.getppid()}_{port}_{''.join(ch for ch in run_id if ch.isalnum())[:32]}"


class Communicator:
    """One rank's endpoint. Collectives are asynchronous on the given (or current) CUDA stream and must be
    issued in the same order on every rank."""

    def __init__(self, handle: int, owner: bool = True) -> None:
        self._h = ctypes.c_void_p(handle)
        self._owner = owner
        L = N.lib()
        self.rank = L.b2_comm_rank(self._h)
        self.world = L.b2_comm_world(self._h)
        self.device = L.b2_comm_device(self._h)
        # The stream every collective of this communicator is issued on while an owner has one (the mini-DDP's comm stream:
        # its bucket allreduces run there during backward).  A caller issuing another collective mid-backward enqueues it on
        # this stream, between event waits in both directions, so the communicator stays one stream-ordered sequence.
        self.ordered_stream: Optional[torch.cuda.Stream] = None

    # ---- construction --------------------------------------------------------------------------
    @classmethod
    def from_env(cls, stage_mb: int = 0, timeout_s: float = 120.0) -> "Communicator":
        """Bootstrap from the env contract torchrun / local_cuda give every worker
        (torch/distributed/elastic/agent/server/local_elastic_agent.py:309-323)."""
        rank = int(os.environ.get("RANK", "0"))
        world = int(os.environ.get("WORLD_SIZE", "1"))
        local_rank = int(os.environ.get("LOCAL_RANK", str(rank)))
        device = int(os.environ.get("B2_DEVICE", str(local_rank)))
        epoch = int(os.environ.get("B2_EPOCH", os.environ.get("TORCHELASTIC_RESTART_COUNT", "0")))
        return cls.create(rank, world, device, default_shm_name(), epoch, stage_mb, timeout_s)

    @classmethod
    def create(cls, rank: int, world: int, device: int, shm_name: str, epoch: int = 0, stage_mb: int = 0,
               timeout_s: float = 120.0) -> "Communicator":
        torch.cuda.set_device(device)
        torch.cuda.init()
        out = ctypes.c_void_p()
        N.check(N.lib().b2_comm_create(ctypes.byref(out), rank, world, device, shm_name.encode(), epoch,
                                       stage_mb << 20, int(timeout_s * 1000)))
        return cls(out.value)

    @classmethod
    def create_local(cls, devices: Sequence[int], stage_mb: int = 0) -> List["Communicator"]:
        """All ranks inside this process (tests / single-GPU parity topology)."""
        torch.cuda.init()
        w = len(devices)
        outs = (ctypes.c_void_p * w)()
        devs = (ctypes.c_int * w)(*devices)
        N.check(N.lib().b2_comm_create_local(outs, w, devs, stage_mb << 20))
        return [cls(outs[i]) for i in range(w)]

    def create_group(self, ranks: Sequence[int], stage_mb: int = 0) -> Optional["Communicator"]:
        """A communicator over the ranks ``ranks`` of this one (include/b200ddp.h: b2_comm_create_group), or None on a rank
        outside them.  Every rank of this communicator calls it, in the same order as its other ``create_group`` calls;
        ``ranks`` is increasing, without duplicates, and the same on every rank.  The result's ``rank`` is this rank's index in
        ``ranks`` and its ``ranks`` the list itself, in this communicator's numbering (its own ``ranks`` when it is a group).
        ``stage_mb`` 0 is ``B2_GROUP_STAGE_MB``.  It inherits the device and the in-kernel timeout, not ``set_param`` values."""
        rs = [as_rank(r) for r in ranks]
        if any(r is None for r in rs):
            raise ValueError(f"create_group: ranks {list(ranks)!r} must be integers")
        out = ctypes.c_void_p()
        arr = (ctypes.c_int * max(len(rs), 1))(*rs)
        N.check(N.lib().b2_comm_create_group(ctypes.byref(out), self._h, len(rs), arr, stage_mb << 20))
        if not out.value:
            return None
        g = type(self)(out.value)
        g.ranks = [self.ranks[r] for r in rs]
        return g

    @property
    def ranks(self) -> List[int]:
        """The global ranks of this communicator, by its rank: ``range(world)`` unless it was made by ``create_group``."""
        return self.__dict__.get("_ranks") or list(range(self.world))

    @ranks.setter
    def ranks(self, value: List[int]) -> None:
        self._ranks = list(value)

    def close(self) -> None:
        if self._h and self._owner:
            N.lib().b2_comm_destroy(self._h)
        self._h = ctypes.c_void_p()

    def __enter__(self) -> "Communicator":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    # ---- tuning / health -----------------------------------------------------------------------
    def set_timeout(self, seconds: float) -> None:
        N.check(N.lib().b2_comm_set_timeout_ms(self._h, int(seconds * 1000)))

    def set_max_ctas(self, n: int) -> None:
        N.check(N.lib().b2_comm_set_max_ctas(self._h, n))

    def set_param(self, name: str, value: int) -> None:
        """AUTO thresholds / pipeline chunking, and the op counter of an idle communicator (include/b200ddp.h:
        b2_comm_set_param); same value on every rank."""
        N.check(N.lib().b2_comm_set_param(self._h, name.encode(), int(value)))

    @property
    def caps(self) -> int:
        return int(N.lib().b2_comm_caps(self._h))

    @property
    def has_multicast(self) -> bool:
        """True when every rank's arena is bound into one NVSwitch multicast object (the NVLS algorithm is available)."""
        return bool(self.caps & N.B2_CAP_MULTICAST)

    def check(self) -> None:
        """Raise if any kernel of this communicator timed out waiting for a peer."""
        N.check(N.lib().b2_comm_status(self._h))

    def trace(self, enable: bool, read_ctas: int = 0):
        """Phase-boundary timestamps (ns, %globaltimer) of the last collective: list of 8-tuples per CTA."""
        buf = (ctypes.c_uint64 * (8 * read_ctas))() if read_ctas else None
        N.check(N.lib().b2_comm_trace(self._h, int(enable), buf, read_ctas))
        return [tuple(buf[8 * i: 8 * i + 8]) for i in range(read_ctas)] if buf is not None else []

    @property
    def last_algo(self) -> str:
        """Name of the algorithm the most recent multi-rank allreduce ran (what "auto" resolved to)."""
        k = int(N.lib().b2_comm_last_algo(self._h))
        return {v: n for n, v in ALGOS.items()}.get(k, "none") if k else "none"

    @property
    def op_count(self) -> int:
        """The device op counter (b2_comm_op_count): collectives completed, plus any ``set_param("op_count", v)``.
        Synchronous."""
        return int(N.lib().b2_comm_op_count(self._h))

    @property
    def launches(self) -> int:
        return int(N.lib().b2_comm_launch_count(self._h))

    @property
    def alltoall_max_bytes(self) -> int:
        """The most bytes one rank may send another in one ``alltoall_`` (b2_alltoall_max_bytes)."""
        return int(N.lib().b2_alltoall_max_bytes(self._h))

    @property
    def p2p_eager_bytes(self) -> int:
        """The largest message a ``p2p_`` send completes without its receive having been launched, once the earlier
        messages to that rank have been received (b2_p2p_eager_bytes)."""
        return int(N.lib().b2_p2p_eager_bytes(self._h))

    # ---- collectives ---------------------------------------------------------------------------
    def allreduce_(self, t: torch.Tensor, scale: Optional[float] = None, wire: str = "bf16", algo: str = "auto",
                   stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """In-place ``t <- round(sum_r wire(scale * t_r))``; scale defaults to 1/world (gradient averaging)."""
        self._check_tensor(t)
        N.check(N.lib().b2_allreduce(self._h, ctypes.c_void_p(t.data_ptr()), t.numel(), mode_for(t, wire),
                                     self._scale(scale), ALGOS[algo], _stream_arg(stream, self.device)))
        return t

    def allreduce_gather_(self, out: torch.Tensor, segments, n_segments: int, scale: Optional[float] = None, wire: str = "bf16",
                          algo: str = "auto", stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """``out <- round(sum_r wire(scale * concat(segments_r)))``: the bucket is only written; the input is read
        straight from the tensors the segment table points at (include/b200ddp.h: b2_allreduce_gather).  ``segments`` is a
        ctypes array of ``_native.B2Segment`` (device pointer, begin, end) covering the bucket in order; it is copied into
        the kernel parameters by the call.  A segment whose pointer is ``_native.B2_SEGMENT_ZEROS`` reads as +0.0, here and
        in ``reduce_scatter_gather_`` / ``reduce_scatter_step_``."""
        self._check_tensor(out)
        N.check(N.lib().b2_allreduce_gather(self._h, ctypes.c_void_p(out.data_ptr()), out.numel(), segments, n_segments, mode_for(out, wire),
                                            self._scale(scale), ALGOS[algo], _stream_arg(stream, self.device)))
        return out

    def broadcast_(self, t: torch.Tensor, root: int = 0, stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        self._check_tensor(t)
        N.check(N.lib().b2_broadcast(self._h, ctypes.c_void_p(t.data_ptr()), t.numel() * t.element_size(), root,
                                     _stream_arg(stream, self.device)))
        return t

    def allreduce_op_(self, t: torch.Tensor, op: str = "sum", stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """In-place ``t <- op over ranks of t`` (include/b200ddp.h: b2_allreduce_op).  Integer SUM wraps, MIN / MAX are
        exact; float SUM / AVG are the gradient allreduce with scale 1 / (1/W)."""
        dt, code = dtype_op_for(t.dtype, op)
        self._check_tensor(t)
        N.check(N.lib().b2_allreduce_op(self._h, ctypes.c_void_p(t.data_ptr()), t.numel(), dt, code,
                                        _stream_arg(stream, self.device)))
        return t

    def allgather_(self, out: torch.Tensor, t: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """``out`` (world x the size of ``t``, same dtype) <- every rank's ``t`` in rank order (b2_allgather).  ``t`` may be
        this rank's block of ``out``."""
        check_allgather(self, out, t)
        N.check(N.lib().b2_allgather(self._h, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(t.data_ptr()),
                                     t.numel() * t.element_size(), _stream_arg(stream, self.device)))
        return out

    def reduce_scatter_(self, out: torch.Tensor, t: torch.Tensor, op: str = "sum",
                        stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """``out`` <- block ``rank`` of the ``allreduce_op_`` of ``t`` (world x the size of ``out``, same dtype) over the ranks
        (include/b200ddp.h: b2_reduce_scatter): the same bits that allreduce leaves there, moving only (W-1)/W of ``t``.
        ``out`` may be this rank's block of ``t``."""
        dt, code = check_reduce_scatter(self, out, t, op)
        N.check(N.lib().b2_reduce_scatter(self._h, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(t.data_ptr()), out.numel(), dt,
                                          code, _stream_arg(stream, self.device)))
        return out

    def reduce_(self, t: torch.Tensor, root: int, op: str = "sum", stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """On rank ``root``, in place, ``t <- op over ranks of t``; every other rank's ``t`` is only read (include/b200ddp.h:
        b2_reduce).  The root ends with the bits ``allreduce_op_`` leaves wherever that allreduce sums in rank order (every
        algorithm but NVLS); each rank sends (W-1)/W of ``t`` and only the root takes the reduced slices back in."""
        dt, code = dtype_op_for(t.dtype, op, "reduce_")
        r = as_rank(root)
        if r is None or not 0 <= r < self.world:
            raise ValueError(f"reduce_: root {root!r} is not a rank of a world of {self.world}")
        self._check_tensor(t)
        N.check(N.lib().b2_reduce(self._h, ctypes.c_void_p(t.data_ptr()), t.numel(), dt, code, r,
                                  _stream_arg(stream, self.device)))
        return t

    def reduce_scatter_gather_(self, out: torch.Tensor, segments, n_segments: int, scale: Optional[float] = None,
                               wire: str = "bf16", stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """``out`` (``block`` elements) <- block ``rank`` of ``allreduce_gather_`` over the padded bucket of ``world * block``
        elements the segment table covers (include/b200ddp.h: b2_reduce_scatter_gather): the same bits that allreduce leaves
        there wherever it sums in rank order, moving only (W-1)/W of the wire data.  The gradient shard of the sharded
        mini-DDP."""
        self._check_tensor(out)
        N.check(N.lib().b2_reduce_scatter_gather(self._h, ctypes.c_void_p(out.data_ptr()), out.numel(), segments, n_segments,
                                                 mode_for(out, wire), self._scale(scale),
                                                 _stream_arg(stream, self.device)))
        return out

    def reduce_scatter_step_(self, block: int, segments, n_segments: int, opt, scale: Optional[float] = None,
                             wire: str = "bf16", stream: Optional[torch.cuda.Stream] = None) -> None:
        """``reduce_scatter_gather_`` with the optimizer step fused in (include/b200ddp.h: b2_reduce_scatter_step): the
        reduced block steps this rank's block of the flat fp32 parameter buffer and its optimizer state as ``opt`` (a
        ``_native.B2Optim``) describes them, with the arithmetic of torch's fused SGD / Adam / AdamW.  The overlap mode of
        the sharded mini-DDP."""
        mode = _MODE_FOR.get(("f32", wire))
        if mode is None:
            raise ValueError(f"unsupported wire format {wire!r}")
        N.check(N.lib().b2_reduce_scatter_step(self._h, block, segments, n_segments, mode, self._scale(scale),
                                               ctypes.byref(opt), _stream_arg(stream, self.device)))

    def reduce_scatter_step_bf16_(self, block: int, segments, n_segments: int, opt, param_bf16: torch.Tensor,
                                  scale: Optional[float] = None, stream: Optional[torch.cuda.Stream] = None) -> None:
        """``reduce_scatter_step_`` for a bf16 bucket with fp32 master weights (include/b200ddp.h:
        b2_reduce_scatter_step_bf16): ``opt.param`` is this rank's block of fp32 masters, which the step updates with the
        bf16 reduced gradient; ``param_bf16`` (this rank's ``block`` elements of the bucket's bf16 parameter buffer) is
        written from every stepped master.  The overlap mode of the sharded mini-DDP with ``master_weights=True``."""
        self._check_tensor(param_bf16)
        if param_bf16.dtype != torch.bfloat16 or param_bf16.numel() != block or not param_bf16.is_contiguous():
            raise ValueError(f"param_bf16 must be {block} contiguous bf16 elements, got {param_bf16.numel()} of {param_bf16.dtype}")
        N.check(N.lib().b2_reduce_scatter_step_bf16(self._h, block, segments, n_segments, self._scale(scale), ctypes.byref(opt),
                                                    ctypes.c_void_p(param_bf16.data_ptr()), _stream_arg(stream, self.device)))

    def alltoall_(self, outs: Sequence[torch.Tensor], ins: Sequence[torch.Tensor],
                  stream: Optional[torch.cuda.Stream] = None) -> Sequence[torch.Tensor]:
        """``outs[r]`` <- the ``ins[rank]`` of rank r, bit for bit (include/b200ddp.h: b2_alltoall).  Both are lists of world
        contiguous tensors on this communicator's device, all of one dtype (any dtype: the copy is of bytes), of any sizes;
        ``outs[r]`` must have as many bytes as rank r sends this rank, and one pair of ranks carries at most
        ``alltoall_max_bytes``.  No tensor of ``outs`` may overlap another tensor of either list."""
        check_alltoall(self.world, outs, ins)
        for t in (*outs, *ins):
            self._check_tensor(t)

        def ptrs(ts):
            return (ctypes.c_void_p * self.world)(*(t.data_ptr() for t in ts))

        def sizes(ts):
            return (ctypes.c_size_t * self.world)(*(t.numel() * t.element_size() for t in ts))

        N.check(N.lib().b2_alltoall(self._h, ptrs(outs), sizes(outs), ptrs(ins), sizes(ins),
                                    _stream_arg(stream, self.device)))
        return outs

    def p2p_(self, ops: Sequence, stream: Optional[torch.cuda.Stream] = None) -> None:
        """One batch of point-to-point operations in one launch (include/b200ddp.h: b2_p2p).  ``ops`` is a list of 1..64
        ``("send" | "recv", tensor, peer)``: a send gives the tensor's bytes to rank ``peer``, a recv fills the tensor with the
        next message rank ``peer`` sends this rank, which must have as many bytes.  Messages between two ranks match in issue
        order; the ops of one batch make progress whatever their order.  Tensors are contiguous, on this communicator's
        device, of any dtype; a recv tensor may not overlap any other tensor of the batch."""
        if not 1 <= len(ops) <= N.B2_P2P_MAX_OPS:
            raise ValueError(f"p2p_: needs 1..{N.B2_P2P_MAX_OPS} ops, got {len(ops)}")
        peers = []
        for k, (kind, _, peer) in enumerate(ops):
            if kind not in ("send", "recv"):
                raise ValueError(f"p2p_: op {k} is {kind!r}, not 'send' or 'recv'")
            peers.append(check_peer(k, peer, self.rank, self.world))
        arr = (N.B2P2pOp * len(ops))()
        for k, ((kind, t, _), peer) in enumerate(zip(ops, peers)):
            self._check_tensor(t)
            arr[k] = N.B2P2pOp(peer, int(kind == "send"), t.data_ptr(), t.numel() * t.element_size())
        N.check(N.lib().b2_p2p(self._h, arr, len(ops), _stream_arg(stream, self.device)))

    def batchnorm_stats_(self, mean: torch.Tensor, invstd: torch.Tensor, count: float, running_mean: Optional[torch.Tensor] = None,
                         running_var: Optional[torch.Tensor] = None, *, momentum: float, eps: float,
                         counts_out: Optional[torch.Tensor] = None, stream: Optional[torch.cuda.Stream] = None) -> None:
        """SyncBatchNorm's statistics exchange (b2_batchnorm_stats): in place, ``mean`` / ``invstd`` (fp32, C channels) <-
        the merge of every rank's (mean, invstd, count) with the arithmetic of torch.batch_norm_gather_stats_with_counts;
        ``running_mean`` / ``running_var`` (fp32) updated in place when given; ``counts_out`` (fp32, world elements) <-
        every rank's count in rank order."""
        C = mean.numel()
        given = [(name, t, n) for name, t, n in (("mean", mean, C), ("invstd", invstd, C), ("running_mean", running_mean, C),
                                                 ("running_var", running_var, C), ("counts_out", counts_out, self.world))
                 if t is not None]
        for name, t, _ in given:
            if t.dtype != torch.float32:
                raise TypeError(f"batchnorm_stats_: {name} must be float32, got {t.dtype}")
        for name, t, n in given:
            self._check_tensor(t)
            if t.numel() != n:
                raise ValueError(f"batchnorm_stats_: {name} has {t.numel()} elements, expected {n}")

        def ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
            return ctypes.c_void_p(t.data_ptr() if t is not None else None)

        N.check(N.lib().b2_batchnorm_stats(self._h, ptr(mean), ptr(invstd), ctypes.c_float(count), C, ptr(running_mean),
                                           ptr(running_var), float(momentum), float(eps), ptr(counts_out),
                                           _stream_arg(stream, self.device)))

    def barrier(self, stream: Optional[torch.cuda.Stream] = None) -> None:
        N.check(N.lib().b2_barrier(self._h, _stream_arg(stream, self.device)))

    def _scale(self, scale: Optional[float]) -> ctypes.c_float:
        """The scale argument of a gradient collective: 1/world (gradient averaging) unless given."""
        return ctypes.c_float(1.0 / self.world if scale is None else scale)

    def _check_tensor(self, t: torch.Tensor) -> None:
        if not t.is_cuda or t.device.index != self.device:
            raise ValueError(f"tensor on {t.device}, communicator on cuda:{self.device}")
        if not t.is_contiguous():
            raise ValueError("collectives need a contiguous tensor")


def local_pass_(t: torch.Tensor, scale: float = 1.0, wire: str = "bf16", stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
    """The W == 1 fused cast/scale pass (b2_local_pass) on its own."""
    dev = t.device.index
    N.check(N.lib().b2_local_pass(ctypes.c_void_p(t.data_ptr()), t.numel(), mode_for(t, wire), ctypes.c_float(scale), dev,
                                  _stream_arg(stream, dev)))
    return t
