"""Worker-side helpers, importable from the training script the launcher starts.

Mirror of reference torchx/distributed/__init__.py (local_rank:26, local_cuda_device:57, local_device:70, rank:91,
world_size:109, init_pg:164, on_rank0_first:231, on_local_rank0_first:278): rank/device discovery from the torchrun
environment contract and barrier-ordered critical sections.  Two backends behind the same functions:

  * a ``torch.distributed`` process group, exactly as the reference does (``init_pg("auto")`` -> nccl on GPU hosts, gloo
    otherwise) - this is what config #1 (CPU/gloo) and unmodified TorchX scripts use;
  * ``init_pg("b200")`` - the peer-buffer communicator from ``libb200ddp.so``: no TCP store, no NCCL.  ``barrier`` /
    ``on_rank0_first``, ``all_reduce``, ``all_gather_into_tensor``, ``all_gather``, ``reduce_scatter_tensor``,
    ``reduce_scatter``, ``broadcast``, ``all_to_all_single``, ``all_to_all``, the point-to-point ``send``, ``recv``,
    ``isend``, ``irecv``, ``P2POp`` / ``batch_isend_irecv``, ``gather`` / ``scatter``, ``reduce`` to a root and the object
    collectives ``all_gather_object``, ``broadcast_object_list``, ``gather_object``, ``scatter_object_list``,
    ``send_object_list`` / ``recv_object_list`` then run on that fabric.  The object collectives unpickle what peers send,
    so they trust every peer, as torch's do.  ``new_group``, ``new_subgroups`` and ``new_subgroups_by_enumeration`` make
    ``B200Group``s, each with its own communicator over a subset of the ranks, which every helper takes as ``group=``.
"""
from __future__ import annotations

import os
import pickle
import warnings
from contextlib import contextmanager
from typing import Any, Iterator, List, Optional

import torch
import torch.distributed as dist

from torchx_b200.util.cuda import has_cuda_devices

_COMM: Optional[Any] = None  # torchx_b200.ddp.Communicator when init_pg("b200") was used


def local_rank() -> int:
    """``LOCAL_RANK``; 0 when the launcher did not set it - with a warning if a process group is nevertheless up, because
    then every process of the node would claim device 0 (reference torchx/distributed/__init__.py:26-54)."""
    if "LOCAL_RANK" in os.environ:
        return int(os.environ["LOCAL_RANK"])
    if dist.is_available() and dist.is_initialized():
        warnings.warn("the default torch.distributed process group is initialized but the `LOCAL_RANK` environment variable is "
                      "not set: local_rank() trivially returns 0.  Launch the script with torchx (local_cuda / local_cwd) or "
                      "torchrun, or set `LOCAL_RANK` yourself.")
    return 0


def rank() -> int:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank()
    return int(os.environ.get("RANK", "0")) if _COMM is None else _COMM.rank


def world_size() -> int:
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size()
    return int(os.environ.get("WORLD_SIZE", "1")) if _COMM is None else _COMM.world


def local_cuda_device() -> torch.device:
    """``cuda:$B2_DEVICE`` under ``local_cuda`` (the scheduler pins the device), else ``cuda:$LOCAL_RANK``."""
    return torch.device("cuda", int(os.environ.get("B2_DEVICE", str(local_rank()))))


def local_device() -> torch.device:
    """The device this process should place its model on: ``cuda:<pinned ordinal>`` when the native communicator or an
    nccl or b200 process group is active, ``cpu`` under any other process group; with nothing initialised, ``cuda`` if
    the host has GPUs else ``cpu`` (reference torchx/distributed/__init__.py:70-88)."""
    if _COMM is not None:
        return torch.device("cuda", _COMM.device)
    if dist.is_available() and dist.is_initialized():
        return local_cuda_device() if dist.get_backend() in ("nccl", "b200") else torch.device("cpu")
    return torch.device("cuda") if has_cuda_devices() else torch.device("cpu")


def is_rank0() -> bool:
    return rank() == 0


def is_local_rank0() -> bool:
    return local_rank() == 0


def communicator() -> Any:
    """The process-wide native communicator (``init_pg("b200")`` must have been called)."""
    if _COMM is None:
        raise RuntimeError('no native communicator: call torchx_b200.distributed.init_pg("b200") first')
    return _COMM


def is_torchelastic_launched() -> bool:
    return "TORCHELASTIC_RUN_ID" in os.environ


def init_pg(backend: str = "auto", **kwargs: Any) -> torch.device:
    """Initialise this worker's collective backend and return the device it should use.

    ``auto``: nccl when CUDA devices exist, gloo otherwise (reference behaviour).  When the process was not launched
    by a torchrun-compatible launcher a trivial single-rank group is created so scripts also run with plain ``python``.
    As in the reference the caller selects the returned device (``torch.cuda.set_device`` / ``.to(device)``).
    ``b200``: rendezvous through the ``local_cuda`` scheduler's shm control block and CUDA IPC; no process group.
    """
    global _COMM
    if backend == "b200":
        if _COMM is None:
            from torchx_b200.ddp import Communicator

            _COMM = Communicator.from_env(**kwargs)
        return torch.device("cuda", _COMM.device)
    if backend == "auto":
        # a CUDA build of torch says is_available() on some CPU hosts: ask for actual devices and for NCCL itself
        has_gpu = torch.cuda.is_available() and torch.cuda.device_count() > 0 and dist.is_nccl_available()
        backend = "nccl" if has_gpu else "gloo"
    if is_torchelastic_launched():
        dist.init_process_group(backend=backend, **kwargs)
    else:  # plain `python script.py`: a one-rank group on a free port, so the same script runs either way
        os.environ["MASTER_ADDR"] = "localhost"
        os.environ["MASTER_PORT"] = "0"
        dist.init_process_group(backend=backend, rank=0, world_size=1, **kwargs)
    return local_cuda_device() if backend == "nccl" else torch.device("cpu")


def barrier(group: Any = None) -> None:
    """A host-blocking barrier over the world, or over ``group`` (a ``B200Group``) under ``init_pg("b200")``."""
    if _COMM is not None and not dist.is_initialized():
        comm = _comm_for(group)
        if comm is None:
            return _not_in_group("barrier")
        comm.barrier()
        torch.cuda.current_stream(comm.device).synchronize()
        comm.check()  # a barrier kernel that gave up on a stalled peer must not let this rank into the critical section
    elif dist.is_initialized():
        dist.barrier() if group is None else dist.barrier(group=group)


def _on_fabric() -> bool:
    """The collectives below run on the native communicator: init_pg("b200") and no torch.distributed process group."""
    return _COMM is not None and not dist.is_initialized()


class B200Group:
    """A group of ranks of the native communicator (``new_group``): ``comm`` is its own communicator, whose rank is this
    process's index in ``ranks`` (the members' global ranks, increasing).  Every helper of this module takes it as
    ``group=``; ``src`` / ``dst`` / ``peer`` are then global ranks and ``group_src`` / ``group_dst`` / ``group_peer`` ranks of
    the group, as in torch.distributed."""

    def __init__(self, comm: Any, ranks: List[int]) -> None:
        self.comm = comm
        self.ranks = list(ranks)

    def rank(self) -> int:
        return self.comm.rank

    def size(self) -> int:
        return len(self.ranks)

    def get_group_rank(self, global_rank: Any) -> int:
        from torchx_b200.ddp.comm import as_rank

        r = as_rank(global_rank)
        if r is None or r not in self.ranks:
            raise ValueError(f"Global rank {global_rank!r} is not part of group {self.ranks}")
        return self.ranks.index(r)

    def get_global_rank(self, group_rank: Any) -> int:
        from torchx_b200.ddp.comm import as_rank

        r = as_rank(group_rank)
        if r is None or not 0 <= r < len(self.ranks):
            raise ValueError(f"Group rank {group_rank!r} is not part of group {self.ranks}")
        return self.ranks[r]

    def __repr__(self) -> str:
        return f"B200Group(ranks={self.ranks})"


NON_GROUP_MEMBER = dist.GroupMember.NON_GROUP_MEMBER  # what new_group returns on a rank outside the group, as torch does


def _is_non_member(group: Any) -> bool:
    return type(group) is int and group == NON_GROUP_MEMBER


def new_group(ranks: Optional[List[int]] = None, stage_mb: Optional[int] = None) -> Any:
    """``torch.distributed.new_group`` under ``init_pg("b200")``: a ``B200Group`` over the global ``ranks`` (any order; None
    is every rank) on a member, ``NON_GROUP_MEMBER`` elsewhere.  Every rank calls it, with the same ranks, in the same order
    as its other ``new_group`` calls.  The group's communicator has its own arena of 2 stages of ``stage_mb`` MiB (default
    ``B2_GROUP_STAGE_MB``, DESIGN.md 2.8) and inherits the world's device and in-kernel timeout."""
    if not _on_fabric():
        raise RuntimeError('new_group: needs init_pg("b200") and no torch.distributed process group; with one, use '
                           "torch.distributed.new_group")
    from torchx_b200.ddp.comm import as_rank

    W = _COMM.world
    members = list(range(W)) if ranks is None else [as_rank(r) for r in ranks]
    if any(r is None or not 0 <= r < W for r in members):
        raise ValueError(f"new_group: ranks {list(ranks)!r} must be ranks of the world of {W}")
    members = sorted(members)
    if len(set(members)) != len(members):
        raise ValueError(f"new_group: ranks {members} repeat a rank")
    if not members:
        raise ValueError("new_group: ranks is empty")
    comm = _COMM.create_group(members, stage_mb or 0)
    return NON_GROUP_MEMBER if comm is None else B200Group(comm, members)


def new_subgroups_by_enumeration(ranks_per_subgroup_list: List[List[int]], timeout: Any = None, backend: Any = None,
                                 pg_options: Any = None, group_desc: Any = None) -> Any:
    """``torch.distributed.new_subgroups_by_enumeration``: one ``new_group`` per list, returns ``(the group of this rank or
    None, every group)`` where a group this rank is not in is ``NON_GROUP_MEMBER``.  A rank in two lists is a ValueError.
    ``timeout``, ``backend``, ``pg_options`` and ``group_desc`` are accepted and ignored."""
    if not _on_fabric():
        return dist.new_subgroups_by_enumeration(ranks_per_subgroup_list, timeout=timeout, backend=backend,
                                                 pg_options=pg_options, group_desc=group_desc)
    if ranks_per_subgroup_list is None or len(ranks_per_subgroup_list) == 0:
        raise ValueError("The arg 'ranks_per_subgroup_list' cannot be empty")
    seen = {}
    for ranks in ranks_per_subgroup_list:  # checked before any group is made, so no rank is left in a half-made set
        for r in ranks:
            if r in seen:
                raise ValueError(f"Rank {r} has appeared in both subgroup {seen[r]} and {ranks}")
            seen[r] = ranks
    subgroups, cur = [], None
    for ranks in ranks_per_subgroup_list:
        g = new_group(ranks)
        subgroups.append(g)
        if isinstance(g, B200Group):
            cur = g
    return cur, subgroups


def new_subgroups(group_size: Optional[int] = None, group: Any = None, timeout: Any = None, backend: Any = None,
                  pg_options: Any = None, group_desc: Any = None) -> Any:
    """``torch.distributed.new_subgroups``: the ranks of ``group`` (None: the world) cut into consecutive groups of
    ``group_size`` (default: the CUDA devices of this host), as ``new_subgroups_by_enumeration``."""
    if not _on_fabric():
        return dist.new_subgroups(group_size, group=group, timeout=timeout, backend=backend, pg_options=pg_options,
                                  group_desc=group_desc)
    if group_size is None:
        if not torch.cuda.is_available():
            raise ValueError("Default group size only takes effect when CUDA is available.If your subgroup using a backend "
                             "that does not depend on CUDA,please pass in 'group_size' correctly.")
        group_size = torch.cuda.device_count()
    if group_size <= 0:
        raise ValueError(f"The arg 'group_size' ({group_size}) must be positive")
    if isinstance(group, B200Group):
        ranks = group.ranks
    elif group is None or group is dist.group.WORLD:
        ranks = list(range(_COMM.world))
    else:
        raise NotImplementedError(_NO_SUBGROUPS)
    if len(ranks) < group_size:
        raise ValueError(f"The arg 'group_size' ({group_size}) must not exceed the world size ({len(ranks)})")
    if len(ranks) % group_size != 0:
        raise ValueError(f"The world size ({len(ranks)}) must be divisible by '{group_size=}'")
    return new_subgroups_by_enumeration([ranks[i: i + group_size] for i in range(0, len(ranks), group_size)])


_NO_SUBGROUPS = ("the b200 communicator has no subgroups but the B200Group of torchx_b200.distributed.new_group: pass "
                 "group=None or a B200Group")


def _comm_for(group: Any, async_op: bool = False) -> Any:
    """The communicator a helper runs on: the world's for None / WORLD, the group's for a ``B200Group``, None for
    ``NON_GROUP_MEMBER``.  Any other group, and ``async_op``, are refused."""
    if group is None or group is dist.group.WORLD:
        comm = _COMM
    elif isinstance(group, B200Group):
        comm = group.comm
    elif _is_non_member(group):
        comm = None
    else:
        raise NotImplementedError(_NO_SUBGROUPS)
    if async_op:
        raise NotImplementedError("the b200 communicator has no work handles: collectives are ordered on the current stream")
    return comm


def _check_native_call(group: Any, async_op: bool) -> None:
    if group is not None and group is not dist.group.WORLD:
        raise NotImplementedError("the b200 communicator has no subgroups: pass group=None")
    if async_op:
        raise NotImplementedError("the b200 communicator has no work handles: collectives are ordered on the current stream")


def _not_in_group(op: str, ret: Any = None) -> Any:
    """What torch.distributed does on a rank outside ``group``: warn and return (``_warn_not_in_group``)."""
    warnings.warn(f"Running {op} on global rank {_COMM.rank} which does not belong to the given group.", stacklevel=3)
    return ret


def _group_rank(fn: str, name: str, group: Any, r: Any, group_r: Any, default: Optional[int] = 0) -> Any:
    """The rank of ``group``'s communicator that a helper's ``name`` (a global rank) or ``group_name`` (a group rank)
    names, as torch's ``_canonicalize_group_rank``: both given, a rank outside the group and, on ``NON_GROUP_MEMBER``, any
    global rank are ValueErrors; on ``NON_GROUP_MEMBER`` a group rank is returned unchecked."""
    if r is not None and group_r is not None:
        raise ValueError(f"{fn}: Can't specify both group_{name} ({group_r!r}) and {name} ({r!r})")
    if group_r is not None:
        if _is_non_member(group):
            return group_r
        from torchx_b200.ddp.comm import as_rank

        k = as_rank(group_r)
        if k is None or not 0 <= k < group.comm.world:
            raise ValueError(f"{fn}: group_{name} {group_r!r} is not a rank of a group of {group.comm.world}")
        return k
    if r is None:
        if default is None:
            raise ValueError(f"{fn}: {name} or group_{name} must be given")
        r = default
    if _is_non_member(group):
        raise ValueError(f"{fn}: {name} {r!r} is a global rank, and this rank is not a member of the group to translate it")
    return group.get_group_rank(r)


def _world_rank(r: Any, group_r: Any) -> Any:
    """``src`` / ``dst`` / ``peer`` on the world, where ``group_src`` ... is the same rank and may stand in for it."""
    if group_r is None:
        return r
    if r is not None and r != group_r:
        raise ValueError(f"group rank {group_r!r} differs from rank {r!r}; the world's group ranks are its ranks")
    return group_r


def _given(**kw: Any) -> dict:
    """The keyword arguments that were given: a call delegated to torch.distributed passes the group_* ranks only then."""
    return {k: v for k, v in kw.items() if v is not None}


def _is_group(group: Any) -> bool:
    return isinstance(group, B200Group) or _is_non_member(group)


_REDUCE_OPS = ((dist.ReduceOp.SUM, "sum"), (dist.ReduceOp.AVG, "avg"), (dist.ReduceOp.MIN, "min"), (dist.ReduceOp.MAX, "max"))


def reduce_op_name(op: Any) -> str:
    """The allreduce_op_ name of a ``torch.distributed.ReduceOp``; ValueError for PRODUCT, the bitwise ops and the rest."""
    for r, name in _REDUCE_OPS:
        if op == r:
            return name
    raise ValueError(f"a reduction on the b200 communicator supports SUM, AVG, MIN and MAX, not {op}")


def all_reduce(tensor: torch.Tensor, op: Any = dist.ReduceOp.SUM, group: Any = None, async_op: bool = False) -> Any:
    """``torch.distributed.all_reduce`` in place.  Under ``init_pg("b200")`` it runs on the native communicator on the current
    stream: integer SUM (wrapping) and MIN / MAX are exact, float SUM / AVG are the rank-order fp32 sum (include/b200ddp.h).
    With a process group it is ``torch.distributed.all_reduce``."""
    if not _on_fabric():
        return dist.all_reduce(tensor, op=op, group=group, async_op=async_op)
    comm = _comm_for(group, async_op)
    if comm is None:
        return _not_in_group("all_reduce")
    comm.allreduce_op_(tensor, reduce_op_name(op))
    return None


def all_gather_into_tensor(output_tensor: torch.Tensor, input_tensor: torch.Tensor, group: Any = None,
                           async_op: bool = False) -> Any:
    """``torch.distributed.all_gather_into_tensor``: ``output_tensor`` holds every rank's ``input_tensor`` in rank order
    along its first dimension (or, flat, as world consecutive blocks)."""
    if not _on_fabric():
        return dist.all_gather_into_tensor(output_tensor, input_tensor, group=group, async_op=async_op)
    comm = _comm_for(group, async_op)
    if comm is None:
        return _not_in_group("all_gather_into_tensor")
    comm.allgather_(output_tensor, input_tensor)
    return None


def all_gather(tensor_list: List[torch.Tensor], tensor: torch.Tensor, group: Any = None, async_op: bool = False) -> Any:
    """``torch.distributed.all_gather``: ``tensor_list[r]`` <- rank r's ``tensor``."""
    if not _on_fabric():
        return dist.all_gather(tensor_list, tensor, group=group, async_op=async_op)
    comm = _comm_for(group, async_op)
    if comm is None:
        return _not_in_group("all_gather")
    if len(tensor_list) != comm.world:
        raise ValueError(f"all_gather: tensor_list has {len(tensor_list)} tensors, world size is {comm.world}")
    for t in tensor_list:
        if t.dtype != tensor.dtype or t.numel() != tensor.numel():
            raise ValueError(f"all_gather: every tensor of tensor_list must be {tensor.dtype} with {tensor.numel()} elements")
    flat = torch.empty((comm.world,) + tuple(tensor.shape), dtype=tensor.dtype, device=tensor.device)
    comm.allgather_(flat, tensor.contiguous())
    for r, t in enumerate(tensor_list):
        t.copy_(flat[r].view_as(t))
    return None


def reduce_scatter_tensor(output: torch.Tensor, input: torch.Tensor, op: Any = dist.ReduceOp.SUM, group: Any = None,
                          async_op: bool = False) -> Any:
    """``torch.distributed.reduce_scatter_tensor``: ``input`` holds world blocks of ``output``'s size (along its first
    dimension, or flat); rank r's ``output`` <- the reduction over ranks of block r.  Under ``init_pg("b200")`` that is
    block r of what ``all_reduce`` with the same op leaves, bit for bit, at (W-1)/W of the input's bytes per rank."""
    if not _on_fabric():
        return dist.reduce_scatter_tensor(output, input, op=op, group=group, async_op=async_op)
    comm = _comm_for(group, async_op)
    if comm is None:
        return _not_in_group("reduce_scatter_tensor")
    comm.reduce_scatter_(output, input, reduce_op_name(op))
    return None


def reduce_scatter(output: torch.Tensor, input_list: List[torch.Tensor], op: Any = dist.ReduceOp.SUM, group: Any = None,
                   async_op: bool = False) -> Any:
    """``torch.distributed.reduce_scatter``: rank r's ``output`` <- the reduction over ranks of their ``input_list[r]``."""
    if not _on_fabric():
        return dist.reduce_scatter(output, input_list, op=op, group=group, async_op=async_op)
    comm = _comm_for(group, async_op)
    if comm is None:
        return _not_in_group("reduce_scatter")
    name = reduce_op_name(op)
    if len(input_list) != comm.world:
        raise ValueError(f"reduce_scatter: input_list has {len(input_list)} tensors, world size is {comm.world}")
    for t in input_list:
        if t.dtype != output.dtype or t.numel() != output.numel():
            raise ValueError(f"reduce_scatter: every tensor of input_list must be {output.dtype} with {output.numel()} elements")
    comm.reduce_scatter_(output, torch.cat([t.reshape(-1) for t in input_list]), name)
    return None


def broadcast(tensor: torch.Tensor, src: Optional[int] = None, group: Any = None, async_op: bool = False,
              group_src: Optional[int] = None) -> Any:
    """``torch.distributed.broadcast`` in place: every rank's ``tensor`` <- rank ``src``'s, bit for bit."""
    if not _on_fabric():
        return dist.broadcast(tensor, src, group=group, async_op=async_op, **_given(group_src=group_src))
    comm = _comm_for(group, async_op)
    if _is_group(group):
        root = _group_rank("broadcast", "src", group, src, group_src)
        if comm is None:
            return _not_in_group("broadcast")
    else:
        root = _world_rank(src, group_src)
    comm.broadcast_(tensor, root=root)
    return None


def _split_rows(t: torch.Tensor, sizes: Optional[List[int]], what: str, world: Optional[int] = None) -> List[torch.Tensor]:
    """``t`` cut along its first dimension into world views: ``sizes`` rows each, or evenly when ``sizes`` is None / empty."""
    world = _COMM.world if world is None else world
    if not sizes:
        if t.size(0) % world:
            raise ValueError(f"all_to_all_single: {what} has {t.size(0)} rows, not a multiple of the world size {world}; "
                             f"pass {what}_split_sizes")
        sizes = [t.size(0) // world] * world
    sizes = [int(k) for k in sizes]
    if len(sizes) != world or min(sizes) < 0 or sum(sizes) != t.size(0):
        raise ValueError(f"all_to_all_single: {what}_split_sizes {sizes} must be {world} row counts >= 0 summing to the "
                         f"{t.size(0)} rows of {what}")
    return list(torch.split(t, sizes, dim=0))


def all_to_all_single(output: torch.Tensor, input: torch.Tensor, output_split_sizes: Optional[List[int]] = None,
                      input_split_sizes: Optional[List[int]] = None, group: Any = None, async_op: bool = False) -> Any:
    """``torch.distributed.all_to_all_single``: ``input`` is cut along its first dimension into world blocks (evenly, or by
    ``input_split_sizes``) and block j goes to rank j; rank r's block lands in ``output``'s r-th block (evenly, or by
    ``output_split_sizes``).  Under ``init_pg("b200")`` the blocks are views of the two tensors, so nothing is copied
    besides the exchange itself, and the result is the same bits; one pair of ranks carries at most
    ``communicator().alltoall_max_bytes`` bytes."""
    if not _on_fabric():
        return dist.all_to_all_single(output, input, output_split_sizes=output_split_sizes, input_split_sizes=input_split_sizes,
                                      group=group, async_op=async_op)
    comm = _comm_for(group, async_op)
    if comm is None:
        return _not_in_group("all_to_all_single")
    comm.alltoall_(_split_rows(output, output_split_sizes, "output", comm.world),
                   _split_rows(input, input_split_sizes, "input", comm.world))
    return None


def all_to_all(output_tensor_list: List[torch.Tensor], input_tensor_list: List[torch.Tensor], group: Any = None,
               async_op: bool = False) -> Any:
    """``torch.distributed.all_to_all``: ``output_tensor_list[r]`` <- rank r's ``input_tensor_list[rank]``.  Under
    ``init_pg("b200")`` the tensors are used where they are (contiguous, one dtype), with no packing copy."""
    if not _on_fabric():
        return dist.all_to_all(output_tensor_list, input_tensor_list, group=group, async_op=async_op)
    comm = _comm_for(group, async_op)
    if comm is None:
        return _not_in_group("all_to_all")
    comm.alltoall_(output_tensor_list, input_tensor_list)
    return None


def send(tensor: torch.Tensor, dst: Optional[int] = None, group: Any = None, tag: int = 0,
         group_dst: Optional[int] = None) -> None:
    """``torch.distributed.send``: rank ``dst`` receives ``tensor``'s bytes.  Under ``init_pg("b200")`` it is enqueued on the
    current stream (as NCCL's is) and messages to one rank match that rank's receives in issue order; ``tag`` is accepted
    and ignored, as torch's NCCL backend does."""
    if not _on_fabric():
        return dist.send(tensor, dst, group=group, tag=tag, **_given(group_dst=group_dst))
    comm = _comm_for(group)
    if _is_group(group):
        peer = _group_rank("send", "dst", group, dst, group_dst, default=None)
        if comm is None:
            return _not_in_group("send")
    else:
        peer = _world_rank(dst, group_dst)
    comm.p2p_([("send", tensor, peer)])
    return None


def recv(tensor: torch.Tensor, src: Optional[int] = None, group: Any = None, tag: int = 0,
         group_src: Optional[int] = None) -> int:
    """``torch.distributed.recv``: ``tensor`` <- the next message rank ``src`` sends this rank (it must have as many bytes);
    returns ``src`` (the global rank).  Receiving from any rank (``src=None``) is not available on the fabric."""
    if not _on_fabric():
        return dist.recv(tensor, src, group=group, tag=tag, **_given(group_src=group_src))
    comm = _comm_for(group)
    if comm is None:
        return _not_in_group("irecv", -1)
    if src is None and group_src is None:
        raise NotImplementedError("the b200 communicator cannot receive from any source: pass src")
    if _is_group(group):
        peer = _group_rank("recv", "src", group, src, group_src)
        comm.p2p_([("recv", tensor, peer)])
        return group.get_global_rank(peer)
    src = _world_rank(src, group_src)
    comm.p2p_([("recv", tensor, src)])
    return src


class _P2PWork:
    """The handle of a point-to-point op on the fabric.  The op is enqueued on the stream that was current at the call, so
    later work on that stream is already ordered after it: ``wait()`` returns True at once.  ``is_completed()`` asks
    whether the GPU has finished it."""

    def __init__(self, event: torch.cuda.Event) -> None:
        self._event = event

    def wait(self, timeout: Any = None) -> bool:
        return True

    def is_completed(self) -> bool:
        return self._event.query()


def _p2p_batch(ops: List[Any], comm: Any = None) -> _P2PWork:
    comm = _COMM if comm is None else comm
    comm.p2p_(ops)
    event = torch.cuda.Event()
    event.record(torch.cuda.current_stream(comm.device))
    return _P2PWork(event)


def isend(tensor: torch.Tensor, dst: Optional[int] = None, group: Any = None, tag: int = 0,
          group_dst: Optional[int] = None) -> Any:
    """``torch.distributed.isend``: ``send`` returning a work handle."""
    if not _on_fabric():
        return dist.isend(tensor, dst, group=group, tag=tag, **_given(group_dst=group_dst))
    comm = _comm_for(group)
    if _is_group(group):
        peer = _group_rank("isend", "dst", group, dst, group_dst, default=None)
        if comm is None:
            return _not_in_group("isend")
    else:
        peer = _world_rank(dst, group_dst)
    return _p2p_batch([("send", tensor, peer)], comm)


def irecv(tensor: torch.Tensor, src: Optional[int] = None, group: Any = None, tag: int = 0,
          group_src: Optional[int] = None) -> Any:
    """``torch.distributed.irecv``: ``recv`` returning a work handle."""
    if not _on_fabric():
        return dist.irecv(tensor, src, group=group, tag=tag, **_given(group_src=group_src))
    comm = _comm_for(group)
    if comm is None:
        return _not_in_group("irecv")
    if src is None and group_src is None:
        raise NotImplementedError("the b200 communicator cannot receive from any source: pass src")
    if _is_group(group):
        peer = _group_rank("irecv", "src", group, src, group_src)
    else:
        peer = _world_rank(src, group_src)
    return _p2p_batch([("recv", tensor, peer)], comm)


class P2POp:
    """``torch.distributed.P2POp``: one entry of ``batch_isend_irecv``.  ``op`` is ``isend`` or ``irecv`` (this module's or
    torch.distributed's).  Under ``init_pg("b200")`` it is a plain record, so it needs no process group; with one it is
    ``torch.distributed.P2POp`` itself, built with torch's ``isend`` / ``irecv`` in place of this module's, so a script
    written with ``P2POp(isend, ...)`` runs under either backend.  With a ``B200Group``, ``peer`` is a global rank and
    ``group_peer`` a rank of the group; the record keeps both."""

    def __new__(cls, op: Any, tensor: torch.Tensor, peer: Optional[int] = None, group: Any = None, tag: int = 0,
                group_peer: Optional[int] = None) -> Any:
        if not _on_fabric():
            op = dist.isend if op is isend else (dist.irecv if op is irecv else op)
            return dist.P2POp(op, tensor, peer, group, tag, **_given(group_peer=group_peer))
        if op not in (isend, irecv, dist.isend, dist.irecv):
            raise ValueError("Invalid ``op``. Expected ``op`` to be of type ``torch.distributed.isend`` or ``torch.distributed.irecv``.")
        self = super().__new__(cls)
        self.op, self.tensor, self.group, self.tag = op, tensor, group, tag
        if _is_group(group):
            if _is_non_member(group):  # torch translates the peer at construction, which a non-member cannot
                raise ValueError("P2POp: this rank is not a member of the group, so its peer cannot be translated")
            self.group_peer = _group_rank("P2POp", "peer", group, peer, group_peer, default=None)
            self.peer = group.get_global_rank(self.group_peer)
        else:
            self.peer = _world_rank(peer, group_peer)
            self.group_peer = self.peer
        return self


def batch_isend_irecv(p2p_op_list: List[Any]) -> List[Any]:
    """``torch.distributed.batch_isend_irecv``: every op of the list in ONE launch under ``init_pg("b200")``, one handle per
    op.  A list longer than the fabric's 64 ops is refused rather than split: the ops of one launch cannot wait on each
    other, and split launches could.  All ops name one group, as torch requires."""
    if not _on_fabric():
        return dist.batch_isend_irecv(p2p_op_list)
    from torchx_b200.ddp._native import B2_P2P_MAX_OPS

    if not p2p_op_list:
        raise ValueError("batch_isend_irecv: p2p_op_list is empty")
    if len(p2p_op_list) > B2_P2P_MAX_OPS:
        raise ValueError(f"batch_isend_irecv: {len(p2p_op_list)} ops, the b200 communicator takes at most {B2_P2P_MAX_OPS} "
                         "in one batch")
    group = p2p_op_list[0].group
    ops = []
    for p in p2p_op_list:
        if _is_group(group) or _is_group(p.group):
            if p.group is not group:
                raise ValueError("All ops need to use the same group.")
            comm = _comm_for(group)
            peer = p.group_peer
        else:
            _check_native_call(p.group, False)
            comm = _COMM
            peer = p.peer
        if peer is None:
            raise NotImplementedError("the b200 communicator cannot receive from any source: pass peer")
        ops.append(("send" if p.op in (isend, dist.isend) else "recv", p.tensor, peer))
    work = _p2p_batch(ops, comm)
    return [work] * len(ops)


def _check_rank(name: str, r: Any, world: Optional[int] = None) -> int:
    from torchx_b200.ddp.comm import as_rank

    world = _COMM.world if world is None else world
    k = as_rank(r)
    if k is None or not 0 <= k < world:
        raise ValueError(f"{name} {r!r} is not a rank of a world of {world}")
    return k


def gather(tensor: torch.Tensor, gather_list: Optional[List[torch.Tensor]] = None, dst: Optional[int] = None, group: Any = None,
           async_op: bool = False, group_dst: Optional[int] = None) -> Any:
    """``torch.distributed.gather``: on rank ``dst`` (default 0), ``gather_list[r]`` <- rank r's ``tensor``.  Under
    ``init_pg("b200")`` rank ``dst`` runs one batch of W - 1 receives and copies its own tensor; every other rank runs one
    send."""
    if not _on_fabric():
        return dist.gather(tensor, gather_list, dst=0 if dst is None and group_dst is None else dst, group=group, async_op=async_op,
                           **_given(group_dst=group_dst))
    comm = _comm_for(group, async_op)
    if comm is None:
        return _not_in_group("gather")
    if _is_group(group):
        dst = _group_rank("gather", "dst", group, dst, group_dst)
    else:
        dst = _check_rank("gather: dst", _world_rank(0 if dst is None and group_dst is None else dst, group_dst))
    if comm.rank != dst:
        if gather_list:
            raise ValueError("Argument ``gather_list`` must NOT be specified on non-destination ranks.")
        comm.p2p_([("send", tensor, dst)])
        return None
    if not gather_list:
        raise ValueError("Argument ``gather_list`` must be specified on destination rank.")
    _check_list("gather: gather_list", gather_list, tensor, comm.world)
    if comm.world > 1:
        comm.p2p_([("recv", t, r) for r, t in enumerate(gather_list) if r != dst])
    gather_list[dst].copy_(tensor)
    return None


def scatter(tensor: torch.Tensor, scatter_list: Optional[List[torch.Tensor]] = None, src: Optional[int] = None, group: Any = None,
            async_op: bool = False, group_src: Optional[int] = None) -> Any:
    """``torch.distributed.scatter``: every rank r's ``tensor`` <- ``scatter_list[r]`` of rank ``src`` (default 0).  Under
    ``init_pg("b200")`` rank ``src`` runs one batch of W - 1 sends and copies its own block; every other rank runs one
    receive."""
    if not _on_fabric():
        return dist.scatter(tensor, scatter_list, src=0 if src is None and group_src is None else src, group=group,
                            async_op=async_op, **_given(group_src=group_src))
    comm = _comm_for(group, async_op)
    if _is_group(group):
        src = _group_rank("scatter", "src", group, src, group_src)
        if comm is None:
            return _not_in_group("scatter")
    else:
        src = _check_rank("scatter: src", _world_rank(0 if src is None and group_src is None else src, group_src))
    if comm.rank != src:
        if scatter_list:
            raise ValueError("Argument ``scatter_list`` must NOT be specified on non-source ranks.")
        comm.p2p_([("recv", tensor, src)])
        return None
    if not scatter_list:
        raise ValueError("Argument ``scatter_list`` must be specified on source rank.")
    _check_list("scatter: scatter_list", scatter_list, tensor, comm.world)
    if comm.world > 1:
        comm.p2p_([("send", t, r) for r, t in enumerate(scatter_list) if r != src])
    tensor.copy_(scatter_list[src])
    return None


def _check_list(what: str, tensors: List[torch.Tensor], like: torch.Tensor, world: Optional[int] = None) -> None:
    world = _COMM.world if world is None else world
    if len(tensors) != world:
        raise ValueError(f"{what} has {len(tensors)} tensors, world size is {world}")
    for t in tensors:
        if t.dtype != like.dtype or t.numel() != like.numel():
            raise ValueError(f"{what}: every tensor must be {like.dtype} with {like.numel()} elements")


def reduce(tensor: torch.Tensor, dst: Optional[int] = None, op: Any = dist.ReduceOp.SUM, group: Any = None,
           async_op: bool = False, group_dst: Optional[int] = None) -> Any:
    """``torch.distributed.reduce`` in place: on rank ``dst``, ``tensor`` <- the reduction over ranks of ``tensor``; every
    other rank's ``tensor`` is only read.  Under ``init_pg("b200")`` rank ``dst`` ends with the bits ``all_reduce`` with the
    same op leaves (include/b200ddp.h: b2_reduce), and each rank sends (W-1)/W of the tensor."""
    if not _on_fabric():
        return dist.reduce(tensor, dst, op=op, group=group, async_op=async_op, **_given(group_dst=group_dst))
    comm = _comm_for(group, async_op)
    if _is_group(group):
        dst = _group_rank("reduce", "dst", group, dst, group_dst, default=None)
        if comm is None:
            return _not_in_group("reduce")
    else:
        dst = _check_rank("reduce: dst", _world_rank(dst, group_dst))
    comm.reduce_(tensor, dst, reduce_op_name(op))
    return None


# ---- object collectives ----------------------------------------------------------------------------------------------
# On the fabric each one pickles every object into a uint8 tensor on the communicator's device, exchanges the int64 sizes,
# then the bytes (padded to the largest size where the exchange needs equal blocks), and unpickles on the host: two fabric
# operations and one device-to-host copy per call, as torch's are.  Unpickling runs whatever the bytes say: these calls
# trust every peer, exactly as torch's do.


def _comm_device() -> torch.device:
    return torch.device("cuda", _COMM.device)


def _check_object_call(fn: str, group: Any, device: Any = None) -> torch.device:
    """The device an object collective runs on: the communicator's.  ``group`` must be None, WORLD or a ``B200Group`` (or
    ``NON_GROUP_MEMBER``) and ``device``, if given, the communicator's device: the fabric never moves the exchange
    elsewhere."""
    _comm_for(group)
    here = _comm_device()
    if device is not None:
        d = torch.device(device)
        if d.type == "cuda" and d.index is None:
            d = torch.device("cuda", torch.cuda.current_device())
        if d != here:
            raise ValueError(f"{fn}: device {device} is not the b200 communicator's device {here}")
    return here


def _peer_arg(fn: str, name: str, r: Any, group_r: Any, default: Optional[int] = 0, group: Any = None) -> int:
    """``src`` / ``dst`` of an object collective, as a rank of ``group``'s communicator.  On the world ``group_src`` /
    ``group_dst`` may stand in for it or repeat it (the world's group rank is the rank); on a group see ``_group_rank``."""
    if _is_group(group):
        return _group_rank(fn, name, group, r, group_r, default)
    if group_r is not None:
        if r is not None and r != group_r:
            raise ValueError(f"{fn}: group_{name} {group_r!r} differs from {name} {r!r}; the b200 communicator has no subgroups")
        r = group_r
    if r is None:
        if default is None:
            raise ValueError(f"{fn}: {name} must be given")
        r = default
    return _check_rank(f"{fn}: {name}", r)


def _to_bytes(obj: Any, device: torch.device) -> torch.Tensor:
    data = pickle.dumps(obj)
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).to(device)


def _padded(t: torch.Tensor, size: int) -> torch.Tensor:
    out = torch.zeros(size, dtype=torch.uint8, device=t.device)
    out[: t.numel()] = t
    return out


def _concat_sizes(tensors: List[torch.Tensor], device: torch.device):
    sizes = torch.tensor([t.numel() for t in tensors], dtype=torch.int64).to(device)
    return sizes, (torch.cat(tensors) if len(tensors) != 1 else tensors[0])


def _split_objects(object_list: List[Any], sizes: List[int], data: torch.Tensor) -> None:
    host = data.cpu().numpy().tobytes()
    at = 0
    for i, n in enumerate(sizes):
        object_list[i] = pickle.loads(host[at: at + n])
        at += n


def all_gather_object(object_list: List[Any], obj: Any, group: Any = None) -> None:
    """``torch.distributed.all_gather_object``: ``object_list[r]`` <- rank r's ``obj`` (any picklable object).  Under
    ``init_pg("b200")``: one all-gather of the sizes, one of the padded bytes.  Unpickling trusts every peer."""
    if not _on_fabric():
        return dist.all_gather_object(object_list, obj, group=group)
    device = _check_object_call("all_gather_object", group)
    comm = _comm_for(group)
    if comm is None:
        return _not_in_group("all_gather_object")
    W = comm.world
    mine = _to_bytes(obj, device)
    sizes = torch.empty(W, dtype=torch.int64, device=device)
    comm.allgather_(sizes, torch.tensor([mine.numel()], dtype=torch.int64).to(device))
    sizes = sizes.tolist()
    block = max(sizes)
    out = torch.empty(W * block, dtype=torch.uint8, device=device)
    comm.allgather_(out, _padded(mine, block))
    host = out.cpu().numpy().tobytes()
    for r in range(W):
        object_list[r] = pickle.loads(host[r * block: r * block + sizes[r]])
    return None


def gather_object(obj: Any, object_gather_list: Optional[List[Any]] = None, dst: Optional[int] = None, group: Any = None,
                  group_dst: Optional[int] = None) -> None:
    """``torch.distributed.gather_object``: on rank ``dst`` (default 0), ``object_gather_list[r]`` <- rank r's ``obj``; the
    other ranks pass no list.  Under ``init_pg("b200")``: an all-gather of the sizes, then ``gather`` of the padded bytes.
    Unpickling trusts every peer."""
    if not _on_fabric():
        return dist.gather_object(obj, object_gather_list, dst=dst, group=group, group_dst=group_dst)
    device = _check_object_call("gather_object", group)
    comm = _comm_for(group)
    dst = _peer_arg("gather_object", "dst", dst, group_dst, group=group)
    if comm is None:
        return _not_in_group("gather_object")
    if comm.rank == dst and not object_gather_list:
        raise ValueError("Argument ``gather_list`` must be specified on destination rank.")
    if comm.rank != dst and object_gather_list:
        raise ValueError("Argument ``gather_list`` must NOT be specified on non-destination ranks.")
    W = comm.world
    mine = _to_bytes(obj, device)
    sizes = torch.empty(W, dtype=torch.int64, device=device)
    comm.allgather_(sizes, torch.tensor([mine.numel()], dtype=torch.int64).to(device))
    sizes = sizes.tolist()
    block = max(sizes)
    grp = group if _is_group(group) else None
    if comm.rank != dst:
        gather(_padded(mine, block), None, group=grp, group_dst=dst)
        return None
    out = torch.empty(W, block, dtype=torch.uint8, device=device)
    gather(_padded(mine, block), list(out.unbind(0)), group=grp, group_dst=dst)
    host = out.cpu().numpy().tobytes()
    for r in range(W):
        object_gather_list[r] = pickle.loads(host[r * block: r * block + sizes[r]])
    return None


def broadcast_object_list(object_list: List[Any], src: Optional[int] = None, group: Any = None, device: Any = None,
                          group_src: Optional[int] = None) -> None:
    """``torch.distributed.broadcast_object_list``: every rank's ``object_list`` (of one length on every rank) <- rank
    ``src``'s (default 0), in place; ``src``'s list is left as it is.  Under ``init_pg("b200")``: one broadcast of the
    sizes, one of the concatenated bytes.  Unpickling trusts rank ``src``."""
    if not _on_fabric():
        return dist.broadcast_object_list(object_list, src=src, group=group, device=device, group_src=group_src)
    dev = _check_object_call("broadcast_object_list", group, device)
    comm = _comm_for(group)
    src = _peer_arg("broadcast_object_list", "src", src, group_src, group=group)
    if comm is None:
        return _not_in_group("broadcast_object_list")
    if comm.rank == src:
        sizes, data = _concat_sizes([_to_bytes(o, dev) for o in object_list], dev)
        comm.broadcast_(sizes, root=src)
        comm.broadcast_(data, root=src)
        return None
    sizes = torch.empty(len(object_list), dtype=torch.int64, device=dev)
    comm.broadcast_(sizes, root=src)
    sizes = sizes.tolist()
    data = torch.empty(sum(sizes), dtype=torch.uint8, device=dev)
    comm.broadcast_(data, root=src)
    _split_objects(object_list, sizes, data)
    return None


def scatter_object_list(scatter_object_output_list: List[Any], scatter_object_input_list: Optional[List[Any]] = None,
                        src: Optional[int] = None, group: Any = None, group_src: Optional[int] = None) -> None:
    """``torch.distributed.scatter_object_list``: every rank r's ``scatter_object_output_list[0]`` <- rank ``src``'s
    (default 0) ``scatter_object_input_list[r]``.  Under ``init_pg("b200")``: one broadcast of the W sizes, then
    ``scatter`` of the padded bytes.  Unpickling trusts rank ``src``."""
    if not _on_fabric():
        return dist.scatter_object_list(scatter_object_output_list, scatter_object_input_list, src=src, group=group,
                                        group_src=group_src)
    device = _check_object_call("scatter_object_list", group)
    comm = _comm_for(group)
    src = _peer_arg("scatter_object_list", "src", src, group_src, group=group)
    if comm is None:
        return _not_in_group("scatter_object_list")
    if not isinstance(scatter_object_output_list, list) or len(scatter_object_output_list) < 1:
        raise ValueError("Expected argument scatter_object_output_list to be a list of size at least 1.")
    W = comm.world
    grp = group if _is_group(group) else None
    if comm.rank == src:
        if scatter_object_input_list is None:
            raise ValueError("source rank must provide non-None scatter_object_input_list")
        if len(scatter_object_input_list) != W:
            raise ValueError(f"scatter_object_list: scatter_object_input_list has {len(scatter_object_input_list)} objects, "
                             f"world size is {W}")
        parts = [_to_bytes(o, device) for o in scatter_object_input_list]
        comm.broadcast_(torch.tensor([t.numel() for t in parts], dtype=torch.int64).to(device), root=src)
        block = max(t.numel() for t in parts)
        out = torch.empty(block, dtype=torch.uint8, device=device)
        scatter(out, [_padded(t, block) for t in parts], group=grp, group_src=src)
        n = parts[src].numel()
    else:
        sizes = torch.empty(W, dtype=torch.int64, device=device)
        comm.broadcast_(sizes, root=src)
        sizes = sizes.tolist()
        out = torch.empty(max(sizes), dtype=torch.uint8, device=device)
        scatter(out, None, group=grp, group_src=src)
        n = sizes[comm.rank]
    scatter_object_output_list[0] = pickle.loads(out[:n].cpu().numpy().tobytes())
    return None


def send_object_list(object_list: List[Any], dst: Optional[int] = None, group: Any = None, device: Any = None,
                     group_dst: Optional[int] = None, use_batch: bool = False) -> None:
    """``torch.distributed.send_object_list``: rank ``dst`` receives ``object_list`` with ``recv_object_list``.  Under
    ``init_pg("b200")``: one send of the sizes, one of the concatenated bytes; ``use_batch`` is accepted and ignored."""
    if not _on_fabric():
        return dist.send_object_list(object_list, dst=dst, group=group, device=device, group_dst=group_dst, use_batch=use_batch)
    dev = _check_object_call("send_object_list", group, device)
    comm = _comm_for(group)
    dst = _peer_arg("send_object_list", "dst", dst, group_dst, default=None, group=group)
    if comm is None:
        return _not_in_group("send_object_list")
    sizes, data = _concat_sizes([_to_bytes(o, dev) for o in object_list], dev)
    comm.p2p_([("send", sizes, dst)])
    comm.p2p_([("send", data, dst)])
    return None


def recv_object_list(object_list: List[Any], src: Optional[int] = None, group: Any = None, device: Any = None,
                     group_src: Optional[int] = None, use_batch: bool = False) -> int:
    """``torch.distributed.recv_object_list``: ``object_list`` (as long as the sender's) <- the objects rank ``src`` sends
    with ``send_object_list``, in place; returns ``src`` (the global rank).  Receiving from any rank is not available on the
    fabric.  Unpickling trusts rank ``src``."""
    if not _on_fabric():
        return dist.recv_object_list(object_list, src=src, group=group, device=device, group_src=group_src, use_batch=use_batch)
    dev = _check_object_call("recv_object_list", group, device)
    comm = _comm_for(group)
    if src is None and group_src is None:
        raise NotImplementedError("the b200 communicator cannot receive from any source: pass src")
    src = _peer_arg("recv_object_list", "src", src, group_src, group=group)
    if comm is None:
        return _not_in_group("recv_object_list", -1)
    sizes = torch.empty(len(object_list), dtype=torch.int64, device=dev)
    comm.p2p_([("recv", sizes, src)])
    sizes = sizes.tolist()
    data = torch.empty(sum(sizes), dtype=torch.uint8, device=dev)
    comm.p2p_([("recv", data, src)])
    _split_objects(object_list, sizes, data)
    return group.get_global_rank(src) if isinstance(group, B200Group) else src


@contextmanager
def on_rank0_first() -> Iterator[None]:
    """Run the block on rank 0 first, then on everyone else (download-once patterns)."""
    if rank() != 0:
        barrier()
    try:
        yield
    finally:
        if rank() == 0:
            barrier()


@contextmanager
def on_local_rank0_first() -> Iterator[None]:
    """Single-box topology: local rank 0 == rank 0 of its node; with one node this equals on_rank0_first()."""
    first = local_rank() == 0
    if not first:
        barrier()
    try:
        yield
    finally:
        if first:
            barrier()


# ``dist.init_process_group("b200")``: the native communicator as a torch.distributed backend (_backend.py)
from torchx_b200.distributed._backend import B200ProcessGroup, register_backend  # noqa: E402

register_backend()
