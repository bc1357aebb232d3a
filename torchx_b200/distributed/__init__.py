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
from typing import Any, Callable, Iterator, List, Optional, Tuple

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


def process_communicator(**kwargs: Any) -> Any:
    """The process's one native communicator, ``_COMM``, made with ``Communicator.from_env(**kwargs)`` and stored if there
    is none yet.  ``init_pg("b200")``, ``init_process_group("b200")``, the mini-DDP and ``B200HookState`` all take it from
    here, so whichever comes first makes the communicator (and its multi-GiB arena) the others share."""
    global _COMM
    if _COMM is None:
        from torchx_b200.ddp import Communicator

        _COMM = Communicator.from_env(**kwargs)
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
    if backend == "b200":
        return torch.device("cuda", process_communicator(**kwargs).device)
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
        comm, _ = _resolve("barrier", group)
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
        if not _is_non_member(g):
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
_NO_ANY_SOURCE = "the b200 communicator cannot receive from any source: pass src"
_ANY_SOURCE = object()  # a _resolve default: a receive without src, which the fabric refuses


def _resolve(fn: str, group: Any, async_op: bool = False, name: Optional[str] = None, r: Any = None, group_r: Any = None,
             default: Any = 0, translate_first: bool = True, check: bool = True, world: Any = None) -> Tuple[Any, Any]:
    """The communicator a helper runs on and, with ``name``, its root or peer as a rank of that communicator.

    The communicator: ``world`` (default ``_COMM``) for ``group`` None / WORLD, the group's own for a ``B200Group``, None for
    ``NON_GROUP_MEMBER``; any other group, and ``async_op``, are refused.  The root: ``r`` is the global rank the helper's
    ``name`` argument gives, ``group_r`` its ``group_<name>``; with neither, ``default`` - a rank, None (refused below as
    not a rank) or ``_ANY_SOURCE`` (refused).  On the world ``group_r`` may stand in for ``r`` or repeat it, and the root is
    range-checked unless ``check`` is False (the communicator checks it).  On a group it is translated as torch's
    ``_canonicalize_group_rank`` does: both given, or a rank outside the group, is a ValueError.  On ``NON_GROUP_MEMBER``
    the root is translated first when ``translate_first`` (a global rank is then a ValueError, a group rank is returned
    unchecked), else not at all: torch's helpers differ there."""
    on_group = isinstance(group, B200Group)
    if group is None or group is dist.group.WORLD:
        comm = _COMM if world is None else world
    elif on_group or _is_non_member(group):
        comm, on_group = group.comm if on_group else None, True
    else:
        raise NotImplementedError(_NO_SUBGROUPS)
    if async_op:
        raise NotImplementedError("the b200 communicator has no work handles: collectives are ordered on the current stream")
    if name is None or (comm is None and not translate_first):
        return comm, None
    if on_group and r is not None and group_r is not None:
        raise ValueError(f"{fn}: Can't specify both group_{name} ({group_r!r}) and {name} ({r!r})")
    if not on_group and group_r is not None:
        if r is not None and r != group_r:
            raise ValueError(f"{fn}: group_{name} {group_r!r} differs from {name} {r!r}; the world's group ranks are its ranks")
        r, group_r = group_r, None
    if not on_group and not check:
        return comm, r
    if r is None and group_r is None:
        if default is _ANY_SOURCE:
            raise NotImplementedError(_NO_ANY_SOURCE)
        r = default
    from torchx_b200.ddp.comm import as_rank

    if not on_group:
        k = as_rank(r)
        if k is None or not 0 <= k < comm.world:
            raise ValueError(f"{fn}: {name} {r!r} is not a rank of a world of {comm.world}")
        return comm, k
    if group_r is not None:
        k = as_rank(group_r)
        if comm is not None and (k is None or not 0 <= k < comm.world):
            raise ValueError(f"{fn}: group_{name} {group_r!r} is not a rank of a group of {comm.world}")
        return comm, group_r if comm is None else k
    if comm is None:
        raise ValueError(f"{fn}: {name} {r!r} is a global rank, and this rank is not a member of the group to translate it")
    return comm, group.get_group_rank(r)


def _global_rank(group: Any, k: Any) -> Any:
    """The global rank of rank ``k`` of the communicator ``_resolve`` returned for ``group``."""
    return k if group is None or group is dist.group.WORLD else group.get_global_rank(k)


def _not_in_group(op: str, ret: Any = None) -> Any:
    """What torch.distributed does on a rank outside ``group``: warn and return (``_warn_not_in_group``)."""
    warnings.warn(f"Running {op} on global rank {_COMM.rank} which does not belong to the given group.", stacklevel=3)
    return ret


def _given(**kw: Any) -> dict:
    """The keyword arguments that were given: a call delegated to torch.distributed passes the group_* ranks only then."""
    return {k: v for k, v in kw.items() if v is not None}


def _on(stream: Any) -> dict:
    """The stream keyword of a Communicator call in a ``launch(stream)``: none for None, the current stream."""
    return {} if stream is None else {"stream": stream}


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
    comm, _ = _resolve("all_reduce", group, async_op)
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
    comm, _ = _resolve("all_gather_into_tensor", group, async_op)
    if comm is None:
        return _not_in_group("all_gather_into_tensor")
    comm.allgather_(output_tensor, input_tensor)
    return None


def all_gather(tensor_list: List[torch.Tensor], tensor: torch.Tensor, group: Any = None, async_op: bool = False) -> Any:
    """``torch.distributed.all_gather``: ``tensor_list[r]`` <- rank r's ``tensor``."""
    if not _on_fabric():
        return dist.all_gather(tensor_list, tensor, group=group, async_op=async_op)
    comm, _ = _resolve("all_gather", group, async_op)
    if comm is None:
        return _not_in_group("all_gather")
    _all_gather(comm, tensor_list, tensor.contiguous())(None)
    return None


def _all_gather(comm: Any, tensor_list: List[torch.Tensor], tensor: torch.Tensor) -> Callable[[Any], None]:
    """``all_gather``'s checks on ``comm``, and its ``launch(stream)``: one all-gather into a staging buffer, then a copy
    per rank.  This and the list collectives below serve the helpers (``launch(None)``) and ``B200ProcessGroup``."""
    _check_list("all_gather: tensor_list", tensor_list, tensor, comm.world, "all_gather: every tensor of tensor_list")

    def launch(stream: Any) -> None:
        flat = torch.empty((comm.world,) + tuple(tensor.shape), dtype=tensor.dtype, device=tensor.device)
        comm.allgather_(flat, tensor, **_on(stream))
        for r, t in enumerate(tensor_list):
            t.copy_(flat[r].view_as(t))

    return launch


def reduce_scatter_tensor(output: torch.Tensor, input: torch.Tensor, op: Any = dist.ReduceOp.SUM, group: Any = None,
                          async_op: bool = False) -> Any:
    """``torch.distributed.reduce_scatter_tensor``: ``input`` holds world blocks of ``output``'s size (along its first
    dimension, or flat); rank r's ``output`` <- the reduction over ranks of block r.  Under ``init_pg("b200")`` that is
    block r of what ``all_reduce`` with the same op leaves, bit for bit, at (W-1)/W of the input's bytes per rank."""
    if not _on_fabric():
        return dist.reduce_scatter_tensor(output, input, op=op, group=group, async_op=async_op)
    comm, _ = _resolve("reduce_scatter_tensor", group, async_op)
    if comm is None:
        return _not_in_group("reduce_scatter_tensor")
    comm.reduce_scatter_(output, input, reduce_op_name(op))
    return None


def reduce_scatter(output: torch.Tensor, input_list: List[torch.Tensor], op: Any = dist.ReduceOp.SUM, group: Any = None,
                   async_op: bool = False) -> Any:
    """``torch.distributed.reduce_scatter``: rank r's ``output`` <- the reduction over ranks of their ``input_list[r]``."""
    if not _on_fabric():
        return dist.reduce_scatter(output, input_list, op=op, group=group, async_op=async_op)
    comm, _ = _resolve("reduce_scatter", group, async_op)
    if comm is None:
        return _not_in_group("reduce_scatter")
    _reduce_scatter(comm, output, input_list, reduce_op_name(op))(None)
    return None


def _reduce_scatter(comm: Any, output: torch.Tensor, input_list: List[torch.Tensor], op: str) -> Callable[[Any], None]:
    """``reduce_scatter``'s checks on ``comm``, and its ``launch(stream)``: the list concatenated, then one reduce-scatter."""
    _check_list("reduce_scatter: input_list", input_list, output, comm.world, "reduce_scatter: every tensor of input_list")
    return lambda stream: comm.reduce_scatter_(output, torch.cat([t.reshape(-1) for t in input_list]), op, **_on(stream))


def broadcast(tensor: torch.Tensor, src: Optional[int] = None, group: Any = None, async_op: bool = False,
              group_src: Optional[int] = None) -> Any:
    """``torch.distributed.broadcast`` in place: every rank's ``tensor`` <- rank ``src``'s, bit for bit."""
    if not _on_fabric():
        return dist.broadcast(tensor, src, group=group, async_op=async_op, **_given(group_src=group_src))
    comm, root = _resolve("broadcast", group, async_op, "src", src, group_src, check=False)
    if comm is None:
        return _not_in_group("broadcast")
    comm.broadcast_(tensor, root=root)
    return None


def _split_rows(t: torch.Tensor, sizes: Optional[List[int]], what: str, world: int) -> List[torch.Tensor]:
    """``t`` cut along its first dimension into world views: ``sizes`` rows each, or evenly when ``sizes`` is None / empty."""
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
    comm, _ = _resolve("all_to_all_single", group, async_op)
    if comm is None:
        return _not_in_group("all_to_all_single")
    _all_to_all_single(comm, output, input, output_split_sizes, input_split_sizes)(None)
    return None


def _all_to_all_single(comm: Any, output: torch.Tensor, input: torch.Tensor, output_split_sizes: Optional[List[int]],  # noqa: A002
                       input_split_sizes: Optional[List[int]]) -> Callable[[Any], None]:
    """``all_to_all_single``'s checks on ``comm``, and its ``launch(stream)``: one all-to-all between views of the two."""
    from torchx_b200.ddp.comm import check_alltoall

    outs = _split_rows(output, output_split_sizes, "output", comm.world)
    ins = _split_rows(input, input_split_sizes, "input", comm.world)
    check_alltoall(comm.world, outs, ins)
    return lambda stream: comm.alltoall_(outs, ins, **_on(stream))


def all_to_all(output_tensor_list: List[torch.Tensor], input_tensor_list: List[torch.Tensor], group: Any = None,
               async_op: bool = False) -> Any:
    """``torch.distributed.all_to_all``: ``output_tensor_list[r]`` <- rank r's ``input_tensor_list[rank]``.  Under
    ``init_pg("b200")`` the tensors are used where they are (contiguous, one dtype), with no packing copy."""
    if not _on_fabric():
        return dist.all_to_all(output_tensor_list, input_tensor_list, group=group, async_op=async_op)
    comm, _ = _resolve("all_to_all", group, async_op)
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
    comm, peer = _resolve("send", group, False, "dst", dst, group_dst, default=None)
    if comm is None:
        return _not_in_group("send")
    comm.p2p_([("send", tensor, peer)])
    return None


def recv(tensor: torch.Tensor, src: Optional[int] = None, group: Any = None, tag: int = 0,
         group_src: Optional[int] = None) -> int:
    """``torch.distributed.recv``: ``tensor`` <- the next message rank ``src`` sends this rank (it must have as many bytes);
    returns ``src`` (the global rank).  Receiving from any rank (``src=None``) is not available on the fabric."""
    if not _on_fabric():
        return dist.recv(tensor, src, group=group, tag=tag, **_given(group_src=group_src))
    comm, peer = _resolve("recv", group, False, "src", src, group_src, default=_ANY_SOURCE, translate_first=False)
    if comm is None:
        return _not_in_group("recv", -1)
    comm.p2p_([("recv", tensor, peer)])
    return _global_rank(group, peer)


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


def _p2p_batch(ops: List[Any], comm: Any) -> _P2PWork:
    comm.p2p_(ops)
    event = torch.cuda.Event()
    event.record(torch.cuda.current_stream(comm.device))
    return _P2PWork(event)


def isend(tensor: torch.Tensor, dst: Optional[int] = None, group: Any = None, tag: int = 0,
          group_dst: Optional[int] = None) -> Any:
    """``torch.distributed.isend``: ``send`` returning a work handle."""
    if not _on_fabric():
        return dist.isend(tensor, dst, group=group, tag=tag, **_given(group_dst=group_dst))
    comm, peer = _resolve("isend", group, False, "dst", dst, group_dst, default=None)
    if comm is None:
        return _not_in_group("isend")
    return _p2p_batch([("send", tensor, peer)], comm)


def irecv(tensor: torch.Tensor, src: Optional[int] = None, group: Any = None, tag: int = 0,
          group_src: Optional[int] = None) -> Any:
    """``torch.distributed.irecv``: ``recv`` returning a work handle."""
    if not _on_fabric():
        return dist.irecv(tensor, src, group=group, tag=tag, **_given(group_src=group_src))
    comm, peer = _resolve("irecv", group, False, "src", src, group_src, default=_ANY_SOURCE, translate_first=False)
    if comm is None:
        return _not_in_group("irecv")
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
        comm, self.group_peer = _resolve("P2POp", group, False, "peer", peer, group_peer, default=None, check=False)
        if comm is None:  # torch translates the peer at construction, which a non-member cannot
            raise ValueError("P2POp: this rank is not a member of the group, so its peer cannot be translated")
        self.peer = _global_rank(group, self.group_peer)
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
    comm, ops = None, []
    for p in p2p_op_list:
        c, _ = _resolve("batch_isend_irecv", p.group)
        if ops and c is not comm:
            raise ValueError("All ops need to use the same group.")
        if p.group_peer is None:
            raise NotImplementedError(_NO_ANY_SOURCE)
        comm = c
        ops.append(("send" if p.op in (isend, dist.isend) else "recv", p.tensor, p.group_peer))
    work = _p2p_batch(ops, comm)
    return [work] * len(ops)


def gather(tensor: torch.Tensor, gather_list: Optional[List[torch.Tensor]] = None, dst: Optional[int] = None, group: Any = None,
           async_op: bool = False, group_dst: Optional[int] = None) -> Any:
    """``torch.distributed.gather``: on rank ``dst`` (default 0), ``gather_list[r]`` <- rank r's ``tensor``.  Under
    ``init_pg("b200")`` rank ``dst`` runs one batch of W - 1 receives and copies its own tensor; every other rank runs one
    send."""
    if not _on_fabric():
        return dist.gather(tensor, gather_list, dst=0 if dst is None and group_dst is None else dst, group=group, async_op=async_op,
                           **_given(group_dst=group_dst))
    comm, dst = _resolve("gather", group, async_op, "dst", dst, group_dst, translate_first=False)
    if comm is None:
        return _not_in_group("gather")
    _gather(comm, tensor, gather_list, dst)(None)
    return None


def _gather(comm: Any, tensor: torch.Tensor, gather_list: Optional[List[torch.Tensor]], dst: int) -> Callable[[Any], None]:
    """``gather``'s checks on ``comm``, and its ``launch(stream)``: rank ``dst`` receives W - 1 messages in one batch and
    copies its own tensor; every other rank sends one."""
    _check_root_list(comm.rank == dst, gather_list, "gather_list", "destination")
    if comm.rank != dst:
        return lambda stream: comm.p2p_([("send", tensor, dst)], **_on(stream))
    _check_list("gather: gather_list", gather_list, tensor, comm.world, "gather: gather_list: every tensor")

    def launch(stream: Any) -> None:
        if comm.world > 1:
            comm.p2p_([("recv", t, r) for r, t in enumerate(gather_list) if r != dst], **_on(stream))
        gather_list[dst].copy_(tensor)

    return launch


def scatter(tensor: torch.Tensor, scatter_list: Optional[List[torch.Tensor]] = None, src: Optional[int] = None, group: Any = None,
            async_op: bool = False, group_src: Optional[int] = None) -> Any:
    """``torch.distributed.scatter``: every rank r's ``tensor`` <- ``scatter_list[r]`` of rank ``src`` (default 0).  Under
    ``init_pg("b200")`` rank ``src`` runs one batch of W - 1 sends and copies its own block; every other rank runs one
    receive."""
    if not _on_fabric():
        return dist.scatter(tensor, scatter_list, src=0 if src is None and group_src is None else src, group=group,
                            async_op=async_op, **_given(group_src=group_src))
    comm, src = _resolve("scatter", group, async_op, "src", src, group_src)
    if comm is None:
        return _not_in_group("scatter")
    _scatter(comm, tensor, scatter_list, src)(None)
    return None


def _scatter(comm: Any, tensor: torch.Tensor, scatter_list: Optional[List[torch.Tensor]], src: int) -> Callable[[Any], None]:
    """``scatter``'s checks on ``comm``, and its ``launch(stream)``: rank ``src`` sends W - 1 messages in one batch and
    copies its own block; every other rank receives one."""
    _check_root_list(comm.rank == src, scatter_list, "scatter_list", "source")
    if comm.rank != src:
        return lambda stream: comm.p2p_([("recv", tensor, src)], **_on(stream))
    _check_list("scatter: scatter_list", scatter_list, tensor, comm.world, "scatter: scatter_list: every tensor")

    def launch(stream: Any) -> None:
        if comm.world > 1:
            comm.p2p_([("send", t, r) for r, t in enumerate(scatter_list) if r != src], **_on(stream))
        tensor.copy_(scatter_list[src])

    return launch


def _check_root_list(root: bool, given: Any, name: str, role: str) -> None:
    """The list argument ``name`` is given on the root (the ``role`` rank) and only there, as torch requires."""
    if root and not given:
        raise ValueError(f"Argument ``{name}`` must be specified on {role} rank.")
    if not root and given:
        raise ValueError(f"Argument ``{name}`` must NOT be specified on non-{role} ranks.")


def _check_list(what: str, tensors: List[torch.Tensor], like: torch.Tensor, world: int, every: str) -> None:
    """``tensors`` are world tensors of ``like``'s dtype and size; ``what`` and ``every`` name them in the errors."""
    if len(tensors) != world:
        raise ValueError(f"{what} has {len(tensors)} tensors, world size is {world}")
    for t in tensors:
        if t.dtype != like.dtype or t.numel() != like.numel():
            raise ValueError(f"{every} must be {like.dtype} with {like.numel()} elements")


def reduce(tensor: torch.Tensor, dst: Optional[int] = None, op: Any = dist.ReduceOp.SUM, group: Any = None,
           async_op: bool = False, group_dst: Optional[int] = None) -> Any:
    """``torch.distributed.reduce`` in place: on rank ``dst``, ``tensor`` <- the reduction over ranks of ``tensor``; every
    other rank's ``tensor`` is only read.  Under ``init_pg("b200")`` rank ``dst`` ends with the bits ``all_reduce`` with the
    same op leaves (include/b200ddp.h: b2_reduce), and each rank sends (W-1)/W of the tensor."""
    if not _on_fabric():
        return dist.reduce(tensor, dst, op=op, group=group, async_op=async_op, **_given(group_dst=group_dst))
    comm, dst = _resolve("reduce", group, async_op, "dst", dst, group_dst, default=None)
    if comm is None:
        return _not_in_group("reduce")
    comm.reduce_(tensor, dst, reduce_op_name(op))
    return None


# ---- object collectives ----------------------------------------------------------------------------------------------
# On the fabric each one pickles every object into a uint8 tensor on the communicator's device, exchanges the int64 sizes,
# then the bytes (padded to the largest size where the exchange needs equal blocks), and unpickles on the host: two fabric
# operations and one device-to-host copy per call, as torch's are.  Unpickling runs whatever the bytes say: these calls
# trust every peer, exactly as torch's do.


def _comm_device() -> torch.device:
    return torch.device("cuda", _COMM.device)


def _object_device(fn: str, device: Any = None) -> torch.device:
    """The device an object collective runs on: the communicator's.  ``device``, if given, must be that device: the fabric
    never moves the exchange elsewhere."""
    here = _comm_device()
    if device is not None:
        d = torch.device(device)
        if d.type == "cuda" and d.index is None:
            d = torch.device("cuda", torch.cuda.current_device())
        if d != here:
            raise ValueError(f"{fn}: device {device} is not the b200 communicator's device {here}")
    return here


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


def _load_objects(object_list: List[Any], data: torch.Tensor, sizes: List[int], block: Optional[int] = None) -> None:
    """``object_list[i]`` <- the object pickled in the i-th ``sizes[i]`` bytes of ``data``: packed one after another, or
    each at the start of a padded block of ``block`` bytes."""
    host = data.cpu().numpy().tobytes()
    at = 0
    for i, n in enumerate(sizes):
        object_list[i] = pickle.loads(host[at: at + n])
        at += n if block is None else block


def _exchange_padded(comm: Any, obj: Any, device: torch.device, object_list: Optional[List[Any]],
                     exchange: Callable[[torch.Tensor, int], Optional[torch.Tensor]]) -> None:
    """All-gather every rank's pickled size, then ``exchange(this rank's bytes padded to the largest size, that size)``,
    which returns the W padded blocks in rank order (or None on a rank that receives nothing), unpickled into
    ``object_list``."""
    mine = _to_bytes(obj, device)
    sizes = torch.empty(comm.world, dtype=torch.int64, device=device)
    comm.allgather_(sizes, torch.tensor([mine.numel()], dtype=torch.int64).to(device))
    sizes = sizes.tolist()
    block = max(sizes)
    out = exchange(_padded(mine, block), block)
    if out is not None:
        _load_objects(object_list, out, sizes, block)


def all_gather_object(object_list: List[Any], obj: Any, group: Any = None) -> None:
    """``torch.distributed.all_gather_object``: ``object_list[r]`` <- rank r's ``obj`` (any picklable object).  Under
    ``init_pg("b200")``: one all-gather of the sizes, one of the padded bytes.  Unpickling trusts every peer."""
    if not _on_fabric():
        return dist.all_gather_object(object_list, obj, group=group)
    comm, _ = _resolve("all_gather_object", group)
    device = _object_device("all_gather_object")
    if comm is None:
        return _not_in_group("all_gather_object")

    def exchange(padded: torch.Tensor, block: int) -> torch.Tensor:
        out = torch.empty(comm.world * block, dtype=torch.uint8, device=device)
        comm.allgather_(out, padded)
        return out

    _exchange_padded(comm, obj, device, object_list, exchange)
    return None


def gather_object(obj: Any, object_gather_list: Optional[List[Any]] = None, dst: Optional[int] = None, group: Any = None,
                  group_dst: Optional[int] = None) -> None:
    """``torch.distributed.gather_object``: on rank ``dst`` (default 0), ``object_gather_list[r]`` <- rank r's ``obj``; the
    other ranks pass no list.  Under ``init_pg("b200")``: an all-gather of the sizes, then ``gather`` of the padded bytes.
    Unpickling trusts every peer."""
    if not _on_fabric():
        return dist.gather_object(obj, object_gather_list, dst=dst, group=group, group_dst=group_dst)
    comm, dst = _resolve("gather_object", group, False, "dst", dst, group_dst)
    device = _object_device("gather_object")
    if comm is None:
        return _not_in_group("gather_object")
    _check_root_list(comm.rank == dst, object_gather_list, "gather_list", "destination")

    def exchange(padded: torch.Tensor, block: int) -> Optional[torch.Tensor]:
        out = torch.empty(comm.world, block, dtype=torch.uint8, device=device) if comm.rank == dst else None
        _gather(comm, padded, None if out is None else list(out.unbind(0)), dst)(None)
        return out

    _exchange_padded(comm, obj, device, object_gather_list, exchange)
    return None


def broadcast_object_list(object_list: List[Any], src: Optional[int] = None, group: Any = None, device: Any = None,
                          group_src: Optional[int] = None) -> None:
    """``torch.distributed.broadcast_object_list``: every rank's ``object_list`` (of one length on every rank) <- rank
    ``src``'s (default 0), in place; ``src``'s list is left as it is.  Under ``init_pg("b200")``: one broadcast of the
    sizes, one of the concatenated bytes.  Unpickling trusts rank ``src``."""
    if not _on_fabric():
        return dist.broadcast_object_list(object_list, src=src, group=group, device=device, group_src=group_src)
    comm, src = _resolve("broadcast_object_list", group, False, "src", src, group_src)
    dev = _object_device("broadcast_object_list", device)
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
    _load_objects(object_list, data, sizes)
    return None


def scatter_object_list(scatter_object_output_list: List[Any], scatter_object_input_list: Optional[List[Any]] = None,
                        src: Optional[int] = None, group: Any = None, group_src: Optional[int] = None) -> None:
    """``torch.distributed.scatter_object_list``: every rank r's ``scatter_object_output_list[0]`` <- rank ``src``'s
    (default 0) ``scatter_object_input_list[r]``.  Under ``init_pg("b200")``: one broadcast of the W sizes, then
    ``scatter`` of the padded bytes.  Unpickling trusts rank ``src``."""
    if not _on_fabric():
        return dist.scatter_object_list(scatter_object_output_list, scatter_object_input_list, src=src, group=group,
                                        group_src=group_src)
    comm, src = _resolve("scatter_object_list", group, False, "src", src, group_src)
    device = _object_device("scatter_object_list")
    if comm is None:
        return _not_in_group("scatter_object_list")
    if not isinstance(scatter_object_output_list, list) or len(scatter_object_output_list) < 1:
        raise ValueError("Expected argument scatter_object_output_list to be a list of size at least 1.")
    W = comm.world
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
        _scatter(comm, out, [_padded(t, block) for t in parts], src)(None)
        n = parts[src].numel()
    else:
        sizes = torch.empty(W, dtype=torch.int64, device=device)
        comm.broadcast_(sizes, root=src)
        sizes = sizes.tolist()
        out = torch.empty(max(sizes), dtype=torch.uint8, device=device)
        _scatter(comm, out, None, src)(None)
        n = sizes[comm.rank]
    _load_objects(scatter_object_output_list, out, [n])
    return None


def send_object_list(object_list: List[Any], dst: Optional[int] = None, group: Any = None, device: Any = None,
                     group_dst: Optional[int] = None, use_batch: bool = False) -> None:
    """``torch.distributed.send_object_list``: rank ``dst`` receives ``object_list`` with ``recv_object_list``.  Under
    ``init_pg("b200")``: one send of the sizes, one of the concatenated bytes; ``use_batch`` is accepted and ignored."""
    if not _on_fabric():
        return dist.send_object_list(object_list, dst=dst, group=group, device=device, group_dst=group_dst, use_batch=use_batch)
    if dst is None and group_dst is None:
        raise ValueError("send_object_list: dst must be given")
    comm, dst = _resolve("send_object_list", group, False, "dst", dst, group_dst)
    dev = _object_device("send_object_list", device)
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
    comm, src = _resolve("recv_object_list", group, False, "src", src, group_src, default=_ANY_SOURCE)
    dev = _object_device("recv_object_list", device)
    if comm is None:
        return _not_in_group("recv_object_list", -1)
    sizes = torch.empty(len(object_list), dtype=torch.int64, device=dev)
    comm.p2p_([("recv", sizes, src)])
    sizes = sizes.tolist()
    data = torch.empty(sum(sizes), dtype=torch.uint8, device=dev)
    comm.p2p_([("recv", data, src)])
    _load_objects(object_list, data, sizes)
    return _global_rank(group, src)


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
