"""SyncBatchNorm on the native communicator.

``torch.nn.SyncBatchNorm`` only synchronises when ``torch.distributed.is_initialized()``; under ``init_pg("b200")`` there is
no process group, so it quietly normalises every rank with its own batch statistics.  This subclass runs the same layer
on the fabric instead: the statistics exchange of its forward (``torch/nn/modules/_functions.py``: all_gather of
(mean, invstd, count), the ``count >= 1`` mask, ``batch_norm_gather_stats_with_counts``) is one ``b2_batchnorm_stats``
kernel with no host sync, and the backward's allreduce of (sum_dy, sum_dy_xmu) is ``allreduce_op_(..., "sum")``.  ATen's
``batch_norm_stats``, ``batch_norm_elemt``, ``batch_norm_backward_reduce`` and ``batch_norm_backward_elemt`` do the
compute, as in torch.  With a process group up, or with neither a group nor a communicator, it is torch's module unchanged.
"""
from __future__ import annotations

from typing import Any, Callable

import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch import nn

from torchx_b200 import distributed as _dist


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


class SyncBatchNorm(nn.SyncBatchNorm):
    """``torch.nn.SyncBatchNorm`` that also synchronises under ``init_pg("b200")``.

    On the fabric (``init_pg("b200")`` and no process group), in training with batch statistics and more than one rank,
    the forward's statistics and the backward's gradient sums are exchanged on the native communicator; the result is
    the same bits as torch's SyncBatchNorm forward (DESIGN.md 2.4).  In eval mode or at one rank it falls back to
    ``F.batch_norm`` as torch does.  Off the fabric it is torch's module.  Refused on the fabric: a ``process_group``
    other than the whole world (NotImplementedError), running statistics that are not float32 (TypeError) and a CPU
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
        comm = _dist.communicator()
        need_sync = bn_training and self.training
        if need_sync:
            if self.process_group is not None and self.process_group is not dist.group.WORLD:
                raise NotImplementedError("the b200 communicator has no subgroups: SyncBatchNorm needs process_group=None")
            for name, t in (("running_mean", running_mean), ("running_var", running_var)):
                if t is not None and t.dtype != torch.float32:
                    raise TypeError(f"SyncBatchNorm on the b200 communicator keeps float32 running statistics, {name} is {t.dtype}")
            if input.device.type != "cuda":
                raise ValueError("SyncBatchNorm expected input tensor to be on GPU")
            need_sync = comm.world > 1
        if not need_sync:
            return F.batch_norm(input, running_mean, running_var, self.weight, self.bias, bn_training, exponential_average_factor,
                                self.eps)
        return _FabricSyncBatchNorm.apply(input, self.weight, self.bias, running_mean, running_var, self.eps,
                                          exponential_average_factor, comm)

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
