"""DistributedDataParallel on the H100 peer-buffer fabric: no torch.distributed, no NCCL.

Public surface mirrors ``torch.nn.parallel.DistributedDataParallel`` where the reference path relies on it
(torch/nn/parallel/distributed.py:664-890: rank-0 parameter/buffer broadcast at construction, 25 MiB buckets with
a 1 MiB first bucket, per-forward buffer broadcast, ``no_sync``, ``module.``-prefixed state dict), so a
``dist.ddp``-launched training script swaps one constructor.  Differences that matter for speed:

  * each bucket is reduced by ONE fused kernel (fp32->bf16 cast + 1/W scale + NVSwitch reduction + bf16->fp32)
    on a side stream while backward continues, instead of bf16_compress_hook's 4 launches;
  * zero-copy bucket fill: the kernel reads the gradients straight from the per-parameter tensors autograd produced
    (a device pointer table per bucket) and writes the averaged values into the persistent flat bucket, which
    ``param.grad`` aliases afterwards (gradient_as_bucket_view semantics) - the Reducer's copy-in pass
    (reducer.cpp mark_variable_ready_dense) and its 8 bytes per element are gone;
  * the layout is the steady-state one from iteration 0 (no rebuild pass);
  * the wrapped module's ``nn.BatchNorm2d`` layers become ``torchx_b200.nn.BatchNorm2d``: channels-last bf16 / fp16
    training runs on bandwidth-bound native kernels, every other input on ATen as before (DESIGN.md 2.5).
"""
from __future__ import annotations

import array
import contextlib
import dataclasses
from typing import Dict, Iterator, List, Optional, Set

import torch
from torch import nn

from .bucketing import MIB, BucketSpec, plan_buckets
from . import _native as N
from .comm import Communicator


def _dense_non_overlapping(t: torch.Tensor) -> bool:
    """True if the tensor's elements tile a contiguous block exactly once in SOME dimension order
    (contiguous, channels_last, any permutation)."""
    expected = 1
    for stride, size in sorted((st, sz) for sz, st in zip(t.shape, t.stride()) if sz != 1):
        if stride != expected:
            return False
        expected *= size
    return True


def _view_like(flat_slice: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    if p.is_contiguous() or not _dense_non_overlapping(p):
        return flat_slice.view(p.shape)
    return flat_slice.as_strided(p.shape, p.stride())


def _find_tensors(obj) -> List[torch.Tensor]:
    """The tensors of a forward's output, looked for where torch's DDP looks: tensors, and the items of lists, tuples, dict
    values and dataclass fields, nested."""
    if isinstance(obj, torch.Tensor):
        return [obj]
    if isinstance(obj, (list, tuple)):
        return [t for o in obj for t in _find_tensors(o)]
    if isinstance(obj, dict):
        return [t for o in obj.values() for t in _find_tensors(o)]
    if dataclasses.is_dataclass(obj) and not isinstance(obj, type):
        return [t for f in dataclasses.fields(obj) for t in _find_tensors(getattr(obj, f.name))]
    return []


def _reached_leaves(outputs: List[torch.Tensor]) -> Set[int]:
    """ids of the leaf tensors whose gradient the autograd graph of ``outputs`` accumulates: every AccumulateGrad node
    reachable from their ``grad_fn`` through ``next_functions`` (reducer.cpp search_unused_parameters), plus outputs that
    are themselves leaves requiring a gradient."""
    reached: Set[int] = set()
    stack = []
    for t in outputs:
        if t.grad_fn is not None:
            stack.append(t.grad_fn)
        elif t.requires_grad:
            reached.add(id(t))
    seen = set()
    while stack:
        fn = stack.pop()
        if fn in seen:
            continue
        seen.add(fn)
        leaf = getattr(fn, "variable", None)  # AccumulateGrad
        if leaf is not None:
            reached.add(id(leaf))
        stack.extend(nxt for nxt, _ in fn.next_functions if nxt is not None and nxt not in seen)
    return reached


class _Bucket:
    def __init__(self, spec: BucketSpec, params: List[nn.Parameter], device: torch.device) -> None:
        self.spec = spec
        self.params = params
        self.dtype = params[0].dtype
        self.flat = torch.zeros(spec.numel, dtype=self.dtype, device=device)
        # like the Reducer, give each view the parameter's own (dense) strides so a channels_last weight gets a
        # channels_last gradient view and the bucket's element order is the gradient's memory order
        self.views = [_view_like(self.flat[o : o + n], p) for o, n, p in zip(spec.offsets, spec.numels, params)]
        # strides of the dims that matter (size > 1): two tensors with these equal have the same memory order
        self.view_strides = [tuple(st for st, sz in zip(v.stride(), v.shape) if sz != 1) for v in self.views]
        self.pending = len(params)
        self.ready = False
        self.launched = False
        self.done = torch.cuda.Event()
        # ---- zero-copy fill: the segment table (begin / end fixed, pointers refreshed per iteration: autograd hands out
        # new tensors); it travels in the kernel parameters, so nothing is copied to the device or has to stay alive
        P = len(params)
        self.segments = None
        if P <= N.B2_MAX_SEGMENTS:
            self.segments = (N.B2Segment * P)()
            for i, (o, n) in enumerate(zip(spec.offsets, spec.numels)):
                self.segments[i].begin = o
                self.segments[i].end = o + n
        self.block = 0  # sharded mode (ZeroRedundancyOptimizer): elements of this rank's shard, else 0

    def shard(self, world: int, device: torch.device, grad_shard: bool = True) -> None:
        """Switch to the ZeRO-1 layout: the bucket is padded to world * block elements, the parameters move into one
        persistent flat buffer of that size, and the full-size gradient bucket gives way to this rank's block-sized
        gradient shard.  The pad reads as zero through a last segment that points at a small zero tensor."""
        from .zero import padded_block

        n_el = self.spec.numel
        self.block = padded_block(n_el, world)
        pad = world * self.block - n_el
        self.flat, self.views = None, None  # the reduced gradient exists only as the shard
        self.param_flat = torch.zeros(world * self.block, dtype=self.dtype, device=device)
        with torch.no_grad():
            for o, n, p in zip(self.spec.offsets, self.spec.numels, self.params):
                v = _view_like(self.param_flat[o : o + n], p)  # the parameter's own strides: channels_last stays so
                v.copy_(p.data)
                p.data = v
        # no gradient shard when the optimizer step runs inside the reduce-scatter (overlap_with_ddp)
        self.shard_grad = torch.zeros(self.block, dtype=self.dtype, device=device) if grad_shard else None
        self.pad_zeros = torch.zeros(max(pad, 1), dtype=self.dtype, device=device)

        def table(ranges):
            segs = (N.B2Segment * (len(ranges) + (pad > 0)))()
            for i, (o, n) in enumerate(ranges):
                segs[i].begin, segs[i].end = o, o + n
            if pad:
                segs[-1].src, segs[-1].begin, segs[-1].end = self.pad_zeros.data_ptr(), n_el, n_el + pad
            return segs

        P = len(self.params)
        self.segments = table(list(zip(self.spec.offsets, self.spec.numels))) if P + (pad > 0) <= N.B2_MAX_SEGMENTS else None
        self.copy_segments = table([(0, n_el)])  # the fallback: the gradients copied into one scratch tensor
        self.scratch = None


class DistributedDataParallel(nn.Module):
    find_unused_parameters = False  # the constructor's keyword; a class default, so an instance built without __init__ has it
    _shard_widen = ()  # ZeRO-1 master weights without overlap: (bf16 gradient shard, fp32 block) widened after each backward

    def __init__(
        self,
        module: nn.Module,
        comm: Optional[Communicator] = None,
        bucket_cap_mb: float = 25.0,
        first_bucket_mb: float = 1.0,
        wire: str = "bf16",
        broadcast_buffers: bool = True,
        algo: str = "auto",
        zero_copy: bool = True,
        find_unused_parameters: bool = False,
    ) -> None:
        super().__init__()
        self.module = module
        if comm is None:  # one communicator per process (each owns a multi-GiB arena)
            from torchx_b200.distributed import process_communicator

            comm = process_communicator()
        self.comm = comm
        self.world_size = self.comm.world
        self.wire = wire
        self.algo = algo
        self.zero_copy = zero_copy
        self.broadcast_buffers = broadcast_buffers
        self.require_backward_grad_sync = True
        self.device = torch.device("cuda", self.comm.device)
        self._params = [p for p in module.parameters() if p.requires_grad]
        if not self._params:
            raise RuntimeError("DistributedDataParallel is not needed when a module doesn't have any parameter that requires a gradient.")
        for p in self._params:
            if p.device != self.device:
                raise ValueError(f"parameter on {p.device}, communicator on {self.device}")
        specs = plan_buckets(
            [p.numel() for p in self._params],
            [p.element_size() for p in self._params],
            [str(p.dtype) for p in self._params],
            int(first_bucket_mb * MIB),
            int(bucket_cap_mb * MIB),
        )
        self.buckets = [_Bucket(s, [self._params[i] for i in s.param_indices], self.device) for s in specs]
        self._bucket_of: Dict[int, _Bucket] = {}
        for b in self.buckets:
            for p in b.params:
                self._bucket_of[id(p)] = b
        self._comm_stream = torch.cuda.Stream(device=self.device)
        prev = self.comm.ordered_stream
        if prev is not None:  # collectives already queued on the previous owner's stream (a b200 process group's) run first
            self._comm_stream.wait_stream(prev)
            torch.cuda.current_stream(self.device).wait_stream(prev)
        # bucket allreduces run on this stream mid-backward: other collectives of the communicator (SyncBatchNorm) join it
        self.comm.ordered_stream = self._comm_stream
        self._ready_event = torch.cuda.Event()
        self._next_bucket = 0
        self._callback_queued = False
        self._profile: Optional[list] = None
        self.copied_in_buckets = 0   # buckets that needed the multi-tensor copy-in (zero-copy not applicable), for tests / bench
        self.gathered_buckets = 0    # buckets whose gradients were read in place by the kernel
        self.sharded = False         # ZeRO-1 layout (ZeroRedundancyOptimizer): each rank keeps one block of every bucket
        self._shard_grads: List = []  # (optimizer view, its gradient shard view, parameter): attached after every synced backward
        self._shard_grads_live = False  # the shards hold a reduced gradient that zero_grad() has not cleared
        self._step_in_backward = None  # a ZeroRedundancyOptimizer(overlap_with_ddp=True): each bucket launch steps it
        self._synced_backwards = 0
        # find_unused_parameters (torch's Reducer semantics, DESIGN.md 2.5): the parameters the last synced forward's output
        # does not reach are marked ready at the first gradient hook and contribute zeros; an int32 map of the parameters
        # whose hook fired since the last synced backward is MAX-reduced after the last bucket, and the ones no rank used
        # keep their .grad
        self.find_unused_parameters = find_unused_parameters
        if find_unused_parameters:
            self._index_of = {id(p): i for i, p in enumerate(self._params)}
            self._unused: List[nn.Parameter] = []  # this iteration's, from the graph walk of the synced forward
            self._unused_ids: Set[int] = set()
            self._locally_used = array.array("i", bytes(4 * len(self._params)))
            self._used_dev = torch.zeros(len(self._params), dtype=torch.int32, device=self.device)
            self._used_host = torch.zeros(len(self._params), dtype=torch.int32).pin_memory()
            self._used_event = torch.cuda.Event()
        self._hooks = [p.register_post_accumulate_grad_hook(self._on_grad_ready) for p in self._params]
        # exact nn.BatchNorm2d layers run channels-last bf16 / fp16 training on native kernels, everything else on ATen;
        # torchvision's ResNet blocks run their ReLUs and residual adds inside those kernels
        from torchx_b200.nn.bn2d import convert_batchnorm
        from torchx_b200.nn.resnet import fuse_resnet

        convert_batchnorm(module)
        fuse_resnet(module)
        self._sync_module_states()

    # ---- construction-time / per-forward state sync (reference: distributed.py:881-890, 2176-2243) ----
    def _broadcast_coalesced(self, tensors: List[torch.Tensor], chunk_bytes: int = 250 * MIB) -> None:
        """Rank 0's values -> every rank, coalesced per dtype into flat chunks (logical element order, so
        channels_last and contiguous replicas agree)."""
        if self.world_size == 1 or not tensors:
            return
        from torchx_b200.nn.batchnorm import _ordered

        by_dtype: Dict[torch.dtype, List[torch.Tensor]] = {}
        for t in tensors:
            by_dtype.setdefault(t.dtype, []).append(t)
        for group in by_dtype.values():
            chunks: List[List[torch.Tensor]] = [[]]
            size = 0
            for t in group:
                nbytes = t.numel() * t.element_size()
                if chunks[-1] and size + nbytes > chunk_bytes:
                    chunks.append([])
                    size = 0
                chunks[-1].append(t)
                size += nbytes
            for chunk in chunks:
                flat = torch.cat([t.detach().reshape(-1) for t in chunk])
                # on the ordered stream, after (and before) whatever the communicator already has queued there, e.g. a
                # b200 process group's async collectives the caller has not waited for yet (DESIGN.md 2.7)
                _ordered(self.comm, lambda s, flat=flat: self.comm.broadcast_(flat, root=0, stream=s))
                if self.comm.rank != 0:
                    outs = torch.split(flat, [t.numel() for t in chunk])
                    torch._foreach_copy_([t.detach() for t in chunk], [o.view_as(t) for o, t in zip(outs, chunk)])

    def _sync_module_states(self) -> None:
        self._broadcast_coalesced([p.data for p in self.module.parameters()] + [b.data for b in self.module.buffers()])

    def _sync_buffers(self) -> None:
        if self.broadcast_buffers and self.world_size > 1:
            bufs = [b.data for b in self.module.buffers()]
            if bufs:
                self._broadcast_coalesced(bufs)

    def _check_shardable(self) -> None:
        if self.sharded:
            raise RuntimeError("this DistributedDataParallel is already sharded by a ZeroRedundancyOptimizer")
        if self._synced_backwards:
            raise RuntimeError("ZeroRedundancyOptimizer must be constructed before the model's first backward")

    def _enable_sharding(self, step_in_backward=None) -> None:
        """The ZeRO-1 layout of every bucket (_Bucket.shard); ZeroRedundancyOptimizer's constructor calls it.  With
        ``step_in_backward`` (an overlap_with_ddp optimizer) every bucket launch also steps that optimizer's shard."""
        self._check_shardable()
        for b in self.buckets:
            b.shard(self.world_size, self.device, grad_shard=step_in_backward is None)
        self.sharded = True
        self._step_in_backward = step_in_backward

    # ---- training step -----------------------------------------------------------------------------
    def _reset_reducer_state(self) -> None:
        """What Reducer::prepare_for_backward does: a backward that raised midway (caught OOM, skipped batch) must
        not leave stale counters behind - the engine drops its queued callbacks in that case."""
        self._callback_queued = False
        self._next_bucket = 0
        for b in self.buckets:
            b.pending, b.ready, b.launched = len(b.params), False, False

    def forward(self, *args, **kwargs):
        synced = torch.is_grad_enabled() and self.require_backward_grad_sync
        if synced:
            self._refuse_unused_capture()
            # a kernel that gave up on a stalled peer leaves undefined bucket contents: never train on them
            self.comm.check()
            self._reset_reducer_state()
            self._sync_buffers()
        out = self.module(*args, **kwargs)
        if synced and self.find_unused_parameters:  # not under no_sync, as in torch
            reached = _reached_leaves(_find_tensors(out))
            self._unused = [p for p in self._params if id(p) not in reached]
            self._unused_ids = {id(p) for p in self._unused}
        return out

    @contextlib.contextmanager
    def no_sync(self) -> Iterator[None]:
        """Gradient accumulation: skip the allreduce inside this context (distributed.py:1507-1531)."""
        old, self.require_backward_grad_sync = self.require_backward_grad_sync, False
        try:
            yield
        finally:
            self.require_backward_grad_sync = old

    def _on_grad_ready(self, p: nn.Parameter) -> None:
        if self.find_unused_parameters:
            self._locally_used[self._index_of[id(p)]] = 1  # no_sync backwards count too
        if not self.require_backward_grad_sync:
            return
        if not self._callback_queued:
            self._refuse_unused_capture()  # a backward captured on its own, after an eager forward
            self._callback_queued = True
            torch.autograd.Variable._execution_engine.queue_callback(self._finalize_backward)
            if self.find_unused_parameters:
                for q in self._unused:
                    self._mark_ready(q)
        if self.find_unused_parameters and id(p) in self._unused_ids:
            raise RuntimeError(
                "a parameter that the forward's output does not reach produced a gradient: it was already marked ready as "
                "unused.  Compute the loss only from the DistributedDataParallel output")
        self._mark_ready(p)

    def _refuse_unused_capture(self) -> None:
        """find_unused_parameters needs the host: the backward copies the locally used map from pageable memory and waits
        for its reduction before it knows which .grad to keep.  Neither can be captured in a CUDA graph, so a synced
        forward or backward under capture raises here, before any bucket is launched."""
        if self.find_unused_parameters and torch.cuda.is_current_stream_capturing():
            raise RuntimeError(
                "find_unused_parameters=True cannot run under CUDA graph capture: the parameters no rank used are known "
                "only after a host wait for the reduced used map; capture with find_unused_parameters=False")

    def _mark_ready(self, p: nn.Parameter) -> None:
        b = self._bucket_of[id(p)]
        b.pending -= 1
        if b.pending == 0:
            b.ready = True
            # launch strictly in bucket order so every rank issues the same collective sequence
            while self._next_bucket < len(self.buckets) and self.buckets[self._next_bucket].ready:
                self._launch(self.buckets[self._next_bucket])
                self._next_bucket += 1
            if self.find_unused_parameters and self._next_bucket == len(self.buckets):
                self._reduce_used_map()

    def _reduce_used_map(self) -> None:
        """After the last bucket: MAX of the locally used maps on the comm stream, copied into pinned host memory.  Every
        rank issues it, whether or not it needs the result (_finalize_backward waits only if some parameter is locally
        unused)."""
        with torch.cuda.stream(self._comm_stream):
            # pageable source: the copy has taken the map's bytes when it returns, so the hooks may write it again
            self._used_dev.copy_(torch.frombuffer(self._locally_used, dtype=torch.int32), non_blocking=True)
            self.comm.allreduce_op_(self._used_dev, "max", stream=self._comm_stream)
            self._used_host.copy_(self._used_dev, non_blocking=True)
            self._used_event.record(self._comm_stream)

    def _gatherable(self, b: _Bucket, grads: List[torch.Tensor]) -> bool:
        """The kernel can read a gradient in place when its memory order IS the bucket's element order: same dtype,
        same (dense) strides as the bucket view the parameter's layout produced."""
        dt = b.dtype
        for g, st in zip(grads, b.view_strides):
            if g is None:  # an unused parameter: a zero segment
                continue
            if g.dtype != dt or not g.is_cuda or tuple(s_ for s_, z in zip(g.stride(), g.shape) if z != 1) != st:
                return False
        return True

    def _launch(self, b: _Bucket) -> None:
        grads = []
        for p in b.params:
            g = p.grad
            if g is None and not self.find_unused_parameters:
                raise RuntimeError("a parameter finished backward without a gradient (unused parameters are not supported)")
            grads.append(g)  # None: an unused parameter without a gradient, which contributes zeros
        gather = self.zero_copy and b.segments is not None and self._gatherable(b, grads)
        if self.sharded:
            self._launch_shard(b, grads, gather)
            return
        if not gather:
            src, dst, zeros = [], [], []
            for g, v in zip(grads, b.views):
                if g is None:
                    zeros.append(v)
                elif g.data_ptr() != v.data_ptr():
                    src.append(g)
                    dst.append(v)
            if src:
                torch._foreach_copy_(dst, src)
            if zeros:
                torch._foreach_zero_(zeros)  # the Reducer's bucket_view.zero_()
            self.copied_in_buckets += 1
        else:
            for seg, g in zip(b.segments, grads):
                seg.src = N.B2_SEGMENT_ZEROS if g is None else g.data_ptr()
            self.gathered_buckets += 1
        cur = torch.cuda.current_stream(self.device)
        self._ready_event.record(cur)
        self._comm_stream.wait_event(self._ready_event)
        if self._profile is not None:
            t0 = torch.cuda.Event(enable_timing=True)
            t0.record(self._comm_stream)
        if gather:
            # the gradient tensors stay referenced by p.grad until _finalize_backward has made the compute stream wait for
            # b.done, so the caching allocator cannot hand their memory out before the kernel has read it
            self.comm.allreduce_gather_(b.flat, b.segments, len(b.params), scale=1.0 / self.world_size, wire=self.wire, algo=self.algo,
                                        stream=self._comm_stream)
        else:
            self.comm.allreduce_(b.flat, scale=1.0 / self.world_size, wire=self.wire, algo=self.algo, stream=self._comm_stream)
        b.done.record(self._comm_stream)
        if self._profile is not None:
            t1 = torch.cuda.Event(enable_timing=True)
            t1.record(self._comm_stream)
            self._profile.append((t0, t1, b.spec.numel * 2 * b.flat.element_size()))
        b.launched = True

    def _launch_shard(self, b: _Bucket, grads: List[torch.Tensor], gather: bool) -> None:
        """Sharded mode: reduce-scatter the bucket (padded to W blocks) into this rank's gradient shard, with the wire,
        scale, order and stream of the allreduce.  Its gradients are read in place, or copied into one scratch tensor
        first when they cannot be (more segments than a table holds, another layout, zero_copy=False)."""
        zero = self._step_in_backward
        if zero is not None:
            zero._refuse_capture()
        if self._next_bucket == 0 and zero is not None and zero._stepped_in_backward:
            # the parameters of this rank's blocks already hold the update of the previous backward: a second update
            # before step() all-gathers it would step from a half-updated model.  Raised before any bucket is launched.
            raise RuntimeError(
                "a second synced backward before step(): with overlap_with_ddp=True each synced backward updates the "
                "parameters; call step() after every synced backward, and accumulate micro-batches under no_sync()")
        if self._next_bucket == 0 and self._shard_grads_live:
            # Unsharded, this backward would add into the reduced gradients still in p.grad.  The sharded gradients live
            # only in the shards, which this backward overwrites: refuse rather than drop the earlier micro-batch.  (Raised
            # before any bucket of this backward is launched, on every rank alike.)
            raise RuntimeError(
                "a second synced backward before zero_grad(): the sharded mini-DDP does not accumulate reduced gradients "
                "across synced backwards; call zero_grad() after step(), and accumulate micro-batches under no_sync()")
        if gather:
            segs = b.segments
            for seg, g in zip(segs, grads):
                seg.src = N.B2_SEGMENT_ZEROS if g is None else g.data_ptr()
            self.gathered_buckets += 1
        else:
            b.scratch = torch.empty(b.spec.numel, dtype=b.dtype, device=self.device)
            views = [_view_like(b.scratch[o : o + n], p) for o, n, p in zip(b.spec.offsets, b.spec.numels, b.params)]
            dst = [v for v, g in zip(views, grads) if g is not None]
            if dst:
                torch._foreach_copy_(dst, [g for g in grads if g is not None])
            if len(dst) < len(views):
                torch._foreach_zero_([v for v, g in zip(views, grads) if g is None])
            segs = b.copy_segments
            segs[0].src = b.scratch.data_ptr()
            self.copied_in_buckets += 1
        cur = torch.cuda.current_stream(self.device)
        self._ready_event.record(cur)
        self._comm_stream.wait_event(self._ready_event)
        if self._profile is not None:
            t0 = torch.cuda.Event(enable_timing=True)
            t0.record(self._comm_stream)
        # the gradients (and the scratch copy) stay referenced until _finalize_backward has made the compute stream wait
        if zero is not None and zero.master_weights and b.dtype == torch.bfloat16:  # steps the masters, writes the bf16 block
            self.comm.reduce_scatter_step_bf16_(b.block, segs, len(segs), zero._launch_table(b),
                                                b.param_flat[self.comm.rank * b.block : (self.comm.rank + 1) * b.block],
                                                scale=1.0 / self.world_size, stream=self._comm_stream)
        elif zero is not None:  # hyper-parameters read now: a scheduler stepped after step() reaches the next backward
            self.comm.reduce_scatter_step_(b.block, segs, len(segs), zero._launch_table(b), scale=1.0 / self.world_size,
                                           wire=self.wire, stream=self._comm_stream)
        else:
            self.comm.reduce_scatter_gather_(b.shard_grad, segs, len(segs), scale=1.0 / self.world_size, wire=self.wire,
                                             stream=self._comm_stream)
        b.done.record(self._comm_stream)
        if self._profile is not None:
            t1 = torch.cuda.Event(enable_timing=True)
            t1.record(self._comm_stream)
            self._profile.append((t0, t1, 2 * b.spec.nbytes))
        b.launched = True

    def _finalize_backward(self) -> None:
        self._callback_queued = False
        try:
            if self._next_bucket != len(self.buckets):
                missing = [b.spec.index for b in self.buckets if not b.launched]
                raise RuntimeError(
                    f"backward finished but buckets {missing} never became ready: some parameters received no gradient "
                    + ("although the forward's output reaches them" if self.find_unused_parameters else
                       "(find_unused_parameters is not supported on this path)"))
            unused: Set[int] = set()  # ids of the parameters no rank used: their .grad stays as it was
            if self.find_unused_parameters and not all(self._locally_used):
                self._used_event.synchronize()  # used on every rank when used here: only then is the reduced map needed
                unused = {id(p) for p, u in zip(self._params, self._used_host.tolist()) if not u}
            cur = torch.cuda.current_stream(self.device)
            for b in self.buckets:
                cur.wait_event(b.done)
                if self.sharded:
                    b.scratch = None
                    for p in b.params:
                        p.grad = None  # frees the full-size gradients: the reduced ones exist only as the shards
                else:
                    for p, v in zip(b.params, b.views):
                        if id(p) not in unused:
                            p.grad = v  # gradient_as_bucket_view: the optimizer reads the averaged bucket in place
            for src, dst in self._shard_widen:  # the fp32 gradients the inner optimizer steps the masters with
                dst.copy_(src)
            for v, g, p in self._shard_grads:
                if id(p) not in unused:
                    v.grad = g
            self._shard_grads_live = bool(self._shard_grads)
            if self._step_in_backward is not None:
                self._step_in_backward._stepped_in_backward = True
            self._synced_backwards += 1
            self.comm.check()
        finally:
            self._next_bucket = 0
            for b in self.buckets:
                b.pending, b.ready, b.launched = len(b.params), False, False
            if self.find_unused_parameters:
                self._locally_used = array.array("i", bytes(4 * len(self._params)))
                self._unused, self._unused_ids = [], set()

    # ---- measurement hooks used by bench.py (CUDA events on the comm stream, around every bucket kernel) ----
    def start_profile(self) -> None:
        self._profile = []

    def stop_profile(self) -> dict:
        """Sum of device time and algorithmic bytes (read the gradients once + write the bucket once) over the bucket
        kernels launched since start_profile(), plus the per-bucket-index mean device time."""
        torch.cuda.synchronize(self.device)
        prof, self._profile = self._profile or [], None
        times = [a.elapsed_time(b) * 1e-3 for a, b, _ in prof]
        seconds = sum(times)
        nb = len(self.buckets)
        per_bucket = []
        if prof and len(prof) % nb == 0:
            for i in range(nb):
                ts = times[i::nb]
                per_bucket.append(round(sum(ts) / len(ts) * 1e6, 2))
        name = "k_local_pass (W=1 fused cast/scale pass)" if self.world_size == 1 else "k_pipe / k_oneshot / k_twoshot (fused bucket allreduce)"
        return {"name": name, "launches": len(prof), "seconds": seconds, "alg_bytes": sum(n for _, _, n in prof), "per_bucket_us": per_bucket}

    def bucket_sizes_mib(self) -> List[float]:
        return [round(b.spec.nbytes / MIB, 2) for b in self.buckets]
