"""SyncBatchNorm on the native communicator.

``torch.nn.SyncBatchNorm`` only synchronises when ``torch.distributed.is_initialized()``; under ``init_pg("b200")`` there is
no process group, so it quietly normalises every rank with its own batch statistics.  This subclass runs the same layer
on the fabric instead: the statistics exchange of its forward (``torch/nn/modules/_functions.py``: all_gather of
(mean, invstd, count), the ``count >= 1`` mask, ``batch_norm_gather_stats_with_counts``) is one ``b2_batchnorm_stats``
kernel with no host sync, and the backward's allreduce of (sum_dy, sum_dy_xmu) is ``allreduce_op_(..., "sum")``.  For a
4-D channels-last bf16 input that ``native_eligible`` and ``native_reductions`` accept, the compute around them runs on
BatchNorm2d's native kernels in their SyncBatchNorm forms (``_SyncStats`` / ``_SyncNormalise``); for every other input
ATen's ``batch_norm_stats``, ``batch_norm_elemt``, ``batch_norm_backward_reduce`` and ``batch_norm_backward_elemt`` do it,
as in torch (``_FabricSyncBatchNorm``).  Both give the same bits.  At one rank an eligible input runs BatchNorm2d's native
path, which gives the bits of torch's ``F.batch_norm``.  With a process group up, or with neither a group nor a
communicator, it is torch's module unchanged.
"""
from __future__ import annotations

from typing import Any, Callable, NamedTuple, Optional

import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd.function import once_differentiable

from torchx_b200 import distributed as _dist
from torchx_b200.nn.bn2d import (N, BatchNorm2d, _NativeBatchNorm, _normalise_backward, _ptr, _stream, _workspace, native_eligible,
                                 native_reductions)


def _ordered(comm: Any, launch: Callable[[torch.cuda.Stream], Any]) -> None:
    """Launch a collective on the current stream, or - while a mini-DDP owns the communicator - on its comm stream, where
    the bucket allreduces of this backward run: the comm stream waits for the current stream, the collective is enqueued,
    and the current stream waits for the comm stream (DESIGN.md 2.5)."""
    cur = torch.cuda.current_stream(comm.device)
    s = comm.ordered_stream
    if s is None:
        launch(cur)
        return
    s.wait_stream(cur)
    launch(s)
    cur.wait_stream(s)


class _FabricSyncBatchNorm(torch.autograd.Function):
    """torch's ``SyncBatchNorm`` function with its collectives on the native communicator."""

    @staticmethod
    def forward(ctx, input, weight, bias, running_mean, running_var, eps, momentum, comm):  # noqa: A002
        if not (input.is_contiguous(memory_format=torch.channels_last)
                or input.is_contiguous(memory_format=torch.channels_last_3d)):
            input = input.contiguous()
        if weight is not None:
            weight = weight.contiguous()
        num_channels = input.shape[1]
        if input.numel() > 0:
            mean, invstd = torch.batch_norm_stats(input, eps)
            count = input.numel() // num_channels
        else:  # an empty rank still takes part, with a zero count that the merge leaves out
            mean = torch.zeros(num_channels, dtype=torch.float32, device=input.device)
            invstd = torch.zeros(num_channels, dtype=torch.float32, device=input.device)
            count = 0
        counts = torch.empty(comm.world, dtype=torch.float32, device=input.device)
        _ordered(comm, lambda s: comm.batchnorm_stats_(mean, invstd, float(count), running_mean, running_var, momentum=momentum,
                                                       eps=eps, counts_out=counts, stream=s))
        ctx.save_for_backward(input, weight, mean, invstd, counts.to(torch.int32))
        ctx.comm = comm
        if input.numel() > 0:
            return torch.batch_norm_elemt(input, weight, bias, mean, invstd, eps)
        return torch.empty_like(input)

    @staticmethod
    def backward(ctx, grad_output):
        if not (grad_output.is_contiguous(memory_format=torch.channels_last)
                or grad_output.is_contiguous(memory_format=torch.channels_last_3d)):
            grad_output = grad_output.contiguous()
        saved_input, weight, mean, invstd, count_tensor = ctx.saved_tensors
        comm = ctx.comm
        grad_input = grad_weight = grad_bias = None
        num_channels = saved_input.shape[1]
        if saved_input.numel() > 0:
            sum_dy, sum_dy_xmu, grad_weight, grad_bias = torch.batch_norm_backward_reduce(
                grad_output, saved_input, mean, invstd, weight, ctx.needs_input_grad[0], ctx.needs_input_grad[1],
                ctx.needs_input_grad[2])
            if ctx.needs_input_grad[0]:
                combined = torch.cat([sum_dy, sum_dy_xmu], dim=0)
                _ordered(comm, lambda s: comm.allreduce_op_(combined, "sum", stream=s))
                sum_dy, sum_dy_xmu = torch.split(combined, num_channels)
                if weight is not None and weight.dtype != mean.dtype:
                    weight = weight.to(mean.dtype)
                grad_input = torch.batch_norm_backward_elemt(grad_output, saved_input, mean, invstd, weight, sum_dy, sum_dy_xmu,
                                                             count_tensor)
            if weight is None or not ctx.needs_input_grad[1]:
                grad_weight = None
            if weight is None or not ctx.needs_input_grad[2]:
                grad_bias = None
        elif ctx.needs_input_grad[0]:  # the peers' allreduce needs this rank's (zero) contribution
            combined = torch.zeros(2 * num_channels, dtype=torch.float32, device=saved_input.device)
            _ordered(comm, lambda s: comm.allreduce_op_(combined, "sum", stream=s))
        return grad_input, grad_weight, grad_bias, None, None, None, None, None


def _native_stats(x: torch.Tensor, eps: float):
    """``torch.batch_norm_stats(x, eps)`` on the native kernels (``b2_bn_stats_invstd``): (mean, invstd)."""
    n, c, h, w = x.shape
    dev = x.device
    mean, invstd = (torch.empty(c, dtype=torch.float32, device=dev) for _ in range(2))
    ws, ws_bytes = _workspace(n * h * w, c, dev)
    N.check(N.lib().b2_bn_stats_invstd(x.data_ptr(), n * h * w, c, N.B2_DT_BFLOAT16, mean.data_ptr(), invstd.data_ptr(), float(eps),
                                       _ptr(ws), ws_bytes, dev.index, _stream(dev)))
    return mean, invstd


class _SyncStats(torch.autograd.Function):
    """The first half of a SyncBatchNorm over several ranks, which ``_SyncNormalise`` finishes: this rank's batch statistics
    (``torch.batch_norm_stats``, on the native kernels with ``native``) and the exchange that merges them and updates the
    running statistics.  Returns x itself (autograd hands back an alias) and the merged mean and invstd.  Its backward is
    the ``dx`` pass (the count form of ``batch_norm_backward_elemt``) from the sums ``_SyncNormalise.backward`` allreduced
    and left in ``sums``."""

    @staticmethod
    def forward(ctx, x, weight, running_mean, running_var, momentum, eps, comm, native, sums):
        c = x.shape[1]
        if native:
            mean, invstd = _native_stats(x, eps)
        elif x.numel() > 0:
            mean, invstd = torch.batch_norm_stats(x, eps)
        else:  # an empty rank still takes part, with a zero count that the merge leaves out
            mean, invstd = (torch.zeros(c, dtype=torch.float32, device=x.device) for _ in range(2))
        counts = torch.empty(comm.world, dtype=torch.float32, device=x.device)
        _ordered(comm, lambda s: comm.batchnorm_stats_(mean, invstd, float(x.numel() // c), running_mean, running_var,
                                                       momentum=momentum, eps=eps, counts_out=counts, stream=s))
        ctx.save_for_backward(x, weight, mean, invstd, counts)
        ctx.native, ctx.sums = native, sums
        ctx.mark_non_differentiable(mean, invstd)
        return x, mean, invstd

    @staticmethod
    @once_differentiable
    def backward(ctx, dy, _mean, _invstd):
        x, weight, mean, invstd, counts = ctx.saved_tensors
        if not ctx.sums:  # _SyncNormalise.backward ran no allreduce: x needs no gradient
            return None, None, None, None, None, None, None, None, None
        sum_dy, sum_dy_xmu = ctx.sums.pop()
        dx = None
        if not ctx.needs_input_grad[0] or x.numel() == 0:
            pass
        elif ctx.native:
            n, c, h, w = x.shape
            dev = x.device
            dx = torch.empty_like(x, memory_format=torch.channels_last)
            N.check(N.lib().b2_bn_backward_elemt_counts(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), n * h * w, c, N.B2_DT_BFLOAT16,
                                                        weight.data_ptr(), mean.data_ptr(), invstd.data_ptr(), sum_dy.data_ptr(),
                                                        sum_dy_xmu.data_ptr(), counts.data_ptr(), counts.numel(), dev.index,
                                                        _stream(dev)))
        else:
            if weight is not None and weight.dtype != mean.dtype:
                weight = weight.to(mean.dtype)
            dx = torch.batch_norm_backward_elemt(dy, x, mean, invstd, weight, sum_dy, sum_dy_xmu, counts.to(torch.int32))
        return dx, None, None, None, None, None, None, None, None


class _SyncNormalise(torch.autograd.Function):
    """The normalise of a SyncBatchNorm whose statistics ``_SyncStats`` merged: ``torch.batch_norm_elemt`` with the merged
    invstd, on the native kernels with ``native``, there with ``relu`` also ``relu_(y + residual)`` in the same pass as
    ``BatchNorm2d``'s ``_Normalise``.  Its backward is the backward reduce, into one [2C] buffer of (sum_dy, sum_dy_xmu)
    that is allreduced in place when ``need_dx`` (the input needs a gradient, as torch's function decides); it returns dy
    (also the residual's gradient) and the local weight / bias gradients, and leaves the sums to ``_SyncStats.backward``."""

    @staticmethod
    def forward(ctx, x, residual, weight, bias, mean, invstd, eps, relu, comm, native, need_dx, sums):
        if native:
            n, c, h, w = x.shape
            dev = x.device
            y = torch.empty_like(x, memory_format=torch.channels_last)
            N.check(N.lib().b2_bn_forward_invstd(x.data_ptr(), _ptr(residual), y.data_ptr(), int(relu), n * h * w, c, N.B2_DT_BFLOAT16,
                                                 weight.data_ptr(), bias.data_ptr(), mean.data_ptr(), invstd.data_ptr(), dev.index,
                                                 _stream(dev)))
        else:
            y = torch.batch_norm_elemt(x, weight, bias, mean, invstd, eps) if x.numel() > 0 else torch.empty_like(x)
        ctx.save_for_backward(x, weight, mean, invstd, y if relu else None)
        ctx.comm, ctx.native, ctx.need_dx, ctx.sums = comm, native, need_dx, sums
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        x, weight, mean, invstd, z = ctx.saved_tensors
        c = x.shape[1]
        need_r, need_w, need_b = ctx.needs_input_grad[1:4]
        combined = torch.empty(2 * c, dtype=torch.float32, device=x.device)
        gw = gb = None
        if ctx.native:
            dy, gw, gb = _normalise_backward(grad_output, x, z, mean, invstd, combined[:c], combined[c:])
        else:
            dy = grad_output
            if not (dy.is_contiguous(memory_format=torch.channels_last) or dy.is_contiguous(memory_format=torch.channels_last_3d)):
                dy = dy.contiguous()
            if x.numel() > 0:
                sum_dy, sum_dy_xmu, gw, gb = torch.batch_norm_backward_reduce(dy, x, mean, invstd, weight, ctx.need_dx, need_w, need_b)
                if ctx.need_dx:  # without input_g ATen's general kernel does not form the sums (they come back None)
                    combined = torch.cat([sum_dy, sum_dy_xmu], dim=0)
            else:  # the peers' allreduce needs this rank's (zero) contribution
                combined.zero_()
        if ctx.need_dx:
            _ordered(ctx.comm, lambda s: ctx.comm.allreduce_op_(combined, "sum", stream=s))
            ctx.sums.append((combined[:c], combined[c:]))
        return (dy, dy if need_r else None, gw if need_w else None, gb if need_b else None, None, None, None, None, None, None, None,
                None)


class _Synced(NamedTuple):
    """What ``SyncBatchNorm.batch_stats`` hands to ``normalise`` over several ranks."""
    x: torch.Tensor
    mean: torch.Tensor
    invstd: torch.Tensor
    comm: Any
    native: bool
    need_dx: bool
    sums: list


class SyncBatchNorm(nn.SyncBatchNorm):
    """``torch.nn.SyncBatchNorm`` that also synchronises under ``init_pg("b200")``.

    On the fabric (``init_pg("b200")`` and no process group), in training with batch statistics and more than one rank,
    the forward's statistics and the backward's gradient sums are exchanged on the native communicator; the result is
    the same bits as torch's SyncBatchNorm forward (DESIGN.md 2.4); the compute runs on native kernels where
    ``native_eligible`` and ``native_reductions`` accept the input.  In eval mode or at one rank it falls back to
    ``F.batch_norm`` as torch does (at one rank on ``BatchNorm2d``'s native path where those accept the input, with the same
    bits).  Off the fabric it is torch's module.  With ``process_group`` a ``B200Group``
    (``torchx_b200.distributed.new_group``) the layer synchronises over the group's ranks only.  Refused on the fabric: any
    other ``process_group`` but the whole world (NotImplementedError), running statistics that are not float32 (TypeError) and a CPU
    input (ValueError)."""

    def forward(self, input: torch.Tensor) -> torch.Tensor:  # noqa: A002
        if not _dist._on_fabric():
            return super().forward(input)
        # torch.nn.SyncBatchNorm.forward up to its need_sync test, which asks torch.distributed
        self._check_input_dim(input)
        self._check_non_zero_input_channels(input)
        exponential_average_factor = 0.0 if self.momentum is None else self.momentum
        if self.training and self.track_running_stats:
            if self.num_batches_tracked is None:
                raise AssertionError("num_batches_tracked must not be None")
            self.num_batches_tracked.add_(1)
            if self.momentum is None:  # cumulative moving average: reads the counter back, as torch does
                exponential_average_factor = 1.0 / self.num_batches_tracked.item()
            else:
                exponential_average_factor = self.momentum
        bn_training = True if self.training else (self.running_mean is None) and (self.running_var is None)
        running_mean = self.running_mean if not self.training or self.track_running_stats else None
        running_var = self.running_var if not self.training or self.track_running_stats else None
        need_sync = bn_training and self.training
        if need_sync:
            # a B200Group's communicator: the statistics of the group's ranks only, merged in group-rank order
            comm, _ = _dist._resolve("SyncBatchNorm", self.process_group)
            if comm is None:  # NON_GROUP_MEMBER
                raise NotImplementedError(_dist._NO_SUBGROUPS)
            for name, t in (("running_mean", running_mean), ("running_var", running_var)):
                if t is not None and t.dtype != torch.float32:
                    raise TypeError(f"SyncBatchNorm on the b200 communicator keeps float32 running statistics, {name} is {t.dtype}")
            if input.device.type != "cuda":
                raise ValueError("SyncBatchNorm expected input tensor to be on GPU")
            need_sync = comm.world > 1
        native = native_eligible(self, input) and native_reductions(input)
        if not need_sync:
            if native and self.eps > 0:  # F.batch_norm refuses eps <= 0
                return _NativeBatchNorm.apply(input, self.weight, self.bias, running_mean, running_var, exponential_average_factor,
                                              self.eps)
            return F.batch_norm(input, running_mean, running_var, self.weight, self.bias, bn_training, exponential_average_factor,
                                self.eps)
        if native:
            return self.normalise(self._sync_stats(input, comm, running_mean, running_var, exponential_average_factor, True))
        return _FabricSyncBatchNorm.apply(input, self.weight, self.bias, running_mean, running_var, self.eps,
                                          exponential_average_factor, comm)

    _training_step = BatchNorm2d._training_step

    def _comm(self) -> Optional[Any]:
        """The communicator this layer synchronises over on the fabric, or None (not on the fabric, or not in its group)."""
        if not _dist._on_fabric():
            return None
        try:
            comm, _ = _dist._resolve("SyncBatchNorm", self.process_group)
        except NotImplementedError:
            return None
        return comm

    def _fusable(self) -> bool:
        """True when a fused ResNet block (``torchx_b200.nn.resnet``) may run this layer as ``batch_stats`` / ``normalise``:
        training on the fabric, in its group, with affine parameters, float32 running statistics (or none) and eps > 0 (at
        one rank torch's F.batch_norm refuses eps <= 0).  Nothing here depends on the input, so every rank decides alike."""
        if not (self.training and self.affine and self.eps > 0 and self._comm() is not None):
            return False
        return all(t is None or t.dtype == torch.float32 for t in (self.running_mean, self.running_var))

    def batch_stats(self, input: torch.Tensor):  # noqa: A002
        """The first half of ``self(input)`` in training on the fabric, for a layer where ``_fusable`` holds.  Over several
        ranks: the batch statistics and their exchange, with the running-statistics update, for any input (on the native
        kernels where ``native_eligible`` and ``native_reductions`` accept it, else on ATen's), so that the exchange, and
        the backward's allreduce in ``normalise``'s node, come in the same order on every rank (DESIGN.md 2.5).  At one rank
        ``BatchNorm2d.batch_stats``, for an input those accept.  ``normalise`` finishes the layer."""
        comm = self._comm()
        if comm.world == 1:
            return BatchNorm2d.batch_stats(self, input)
        if input.device.type != "cuda":
            raise ValueError("SyncBatchNorm expected input tensor to be on GPU")
        running_mean, running_var, momentum = self._training_step()
        native = native_eligible(self, input) and native_reductions(input)
        if not native and not (input.is_contiguous(memory_format=torch.channels_last)
                               or input.is_contiguous(memory_format=torch.channels_last_3d)):
            input = input.contiguous()
        return self._sync_stats(input, comm, running_mean, running_var, momentum, native)

    def _sync_stats(self, input, comm, running_mean, running_var, momentum, native) -> _Synced:
        sums = []  # the allreduced sums, from _SyncNormalise.backward to _SyncStats.backward
        x, mean, invstd = _SyncStats.apply(input, self.weight, running_mean, running_var, momentum, self.eps, comm, native, sums)
        return _Synced(x, mean, invstd, comm, native, input.requires_grad, sums)

    def normalise(self, stats, residual: Optional[torch.Tensor] = None, relu: bool = False) -> torch.Tensor:
        """The rest of ``self(input)`` from ``batch_stats(input)``: the output, or with ``relu`` ``relu_(output + residual)``
        (``relu_(output)`` without a residual), the same bits as those ops after the layer.  On the native kernels the
        ReLU and the residual add run in the normalise pass; a residual must then be a bf16 channels-last tensor of the
        input's shape and device, 16-byte aligned."""
        if not isinstance(stats, _Synced):
            return BatchNorm2d.normalise(self, stats, residual, relu)
        if stats.native:
            return _SyncNormalise.apply(stats.x, residual, self.weight, self.bias, stats.mean, stats.invstd, self.eps, relu,
                                        stats.comm, True, stats.need_dx, stats.sums)
        out = _SyncNormalise.apply(stats.x, None, self.weight, self.bias, stats.mean, stats.invstd, self.eps, False, stats.comm,
                                   False, stats.need_dx, stats.sums)
        if residual is not None:
            out += residual
        return torch.relu_(out) if relu else out

    @classmethod
    def convert_sync_batchnorm(cls, module: nn.Module, process_group: Any = None) -> nn.Module:
        """Replace every ``BatchNorm*D`` and every ``torch.nn.SyncBatchNorm`` layer of ``module`` by this class, sharing its
        parameters and buffers (``num_batches_tracked`` included) and copying ``training``, ``requires_grad`` and
        ``qconfig``; the state-dict keys stay the same.  A converted ``module`` itself is returned as the new layer."""
        module_output = module
        if isinstance(module, nn.modules.batchnorm._BatchNorm) and type(module) is not cls:
            module_output = cls(module.num_features, module.eps, module.momentum, module.affine, module.track_running_stats,
                                process_group)
            if module.affine:
                with torch.no_grad():
                    module_output.weight = module.weight
                    module_output.bias = module.bias
            module_output.running_mean = module.running_mean
            module_output.running_var = module.running_var
            module_output.num_batches_tracked = module.num_batches_tracked
            module_output.training = module.training
            if hasattr(module, "qconfig"):
                module_output.qconfig = module.qconfig
        for name, child in module.named_children():
            module_output.add_module(name, cls.convert_sync_batchnorm(child, process_group))
        del module
        return module_output
