"""Training-mode ``BatchNorm2d`` on native sm_90a kernels for channels-last bf16 activations.

ATen's channels-last BatchNorm kernels give each thread one channel and load one 2-byte element at a time.  Here all four
passes read (and write) 16-byte vecs of 8 channels (DESIGN.md 2.3): the forward statistics and the backward reduce
(``b2_bn_stats`` / ``b2_bn_backward_reduce``), which run ATen's reduction tree in ATen's order, and the forward normalise
and backward ``dx`` (``b2_bn_forward_elemt`` / ``b2_bn_backward_elemt``), ATen's expressions.  So every output, gradient
and running statistic is the bits ``nn.BatchNorm2d`` computes (DESIGN.md 2.4).  An input of 2^31 - 1 elements or more keeps
ATen's reduction calls (``torch.batch_norm_update_stats``, ``torch.batch_norm_backward_reduce``), as ATen reduces those on
another path.  fp16 activations stay on ATen: there torch's BatchNorm runs cuDNN's kernels, whose bits these passes do not
reproduce.

``BatchNorm2d.batch_stats`` / ``normalise`` also run the ReLU that follows the layer, and a residual add before it, inside
the normalise and backward-reduce passes (``b2_bn_forward_relu`` / ``b2_bn_backward_reduce_relu``) with the unfused ops' bits;
``torchx_b200.nn.resnet`` uses it for torchvision's ResNet blocks.

``torchx_b200.nn.SyncBatchNorm`` runs the same passes in their SyncBatchNorm forms (``b2_bn_stats_invstd``,
``b2_bn_forward_invstd``, ``b2_bn_backward_elemt_counts``) around its exchanges.

``BatchNorm2d`` is ``nn.BatchNorm2d`` with the same parameters, buffers, state-dict keys and hooks; it takes the native
path only for an input that the kernels cover exactly (``native_eligible``) and calls ``nn.BatchNorm2d.forward``
unchanged for everything else: eval mode, fp32 or NCHW inputs, CPU tensors, non-affine layers, and every input torch
rejects.  ``convert_batchnorm`` switches the layers of a model over in place.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch
from torch import nn
from torch.autograd.function import once_differentiable

from torchx_b200.ddp import _native as N



def _stream(dev: torch.device) -> int:
    return torch.cuda.current_stream(dev).cuda_stream


def _batch_stats(x, running_mean, running_var, momentum):
    """ATen's training forward up to the normalise: batch_norm_mean_var, then the running-statistics update."""
    n, c, h, w = x.shape
    dev = x.device
    if not native_reductions(x):
        return torch.batch_norm_update_stats(x, running_mean, running_var, momentum)
    mean = torch.empty(c, dtype=torch.float32, device=dev)
    var = torch.empty(c, dtype=torch.float32, device=dev)
    ws, ws_bytes = _workspace(n * h * w, c, dev)
    N.check(N.lib().b2_bn_stats(x.data_ptr(), n * h * w, c, N.B2_DT_BFLOAT16, mean.data_ptr(), var.data_ptr(), _ptr(running_mean),
                                _ptr(running_var), float(momentum), _ptr(ws), ws_bytes, dev.index, _stream(dev)))
    return mean, var


def _backward_elemt(dy, x, weight, mean, invstd, sum_dy, sum_dy_xmu):
    """dx of the BatchNorm from the gradient dy of its output and the backward reduce's sums."""
    n, c, h, w = x.shape
    dev = x.device
    dx = torch.empty_like(x, memory_format=torch.channels_last)
    N.check(N.lib().b2_bn_backward_elemt(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), n * h * w, c, N.B2_DT_BFLOAT16, weight.data_ptr(),
                                         mean.data_ptr(), invstd.data_ptr(), sum_dy.data_ptr(), sum_dy_xmu.data_ptr(), dev.index,
                                         _stream(dev)))
    return dx


class _NativeBatchNorm(torch.autograd.Function):
    """Training-mode batch norm of a channels-last [N, C, H, W] bf16 tensor: ATen's ``native_batch_norm`` with its
    passes native.  Saves what ATen saves: the input, the weight and the batch mean / invstd."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, momentum, eps):
        n, c, h, w = x.shape
        dev = x.device
        mean, var = _batch_stats(x, running_mean, running_var, momentum)
        y = torch.empty_like(x, memory_format=torch.channels_last)
        invstd = torch.empty(c, dtype=torch.float32, device=dev)
        N.check(N.lib().b2_bn_forward_elemt(x.data_ptr(), y.data_ptr(), n * h * w, c, N.B2_DT_BFLOAT16, weight.data_ptr(),
                                            bias.data_ptr(), mean.data_ptr(), var.data_ptr(), float(eps), invstd.data_ptr(),
                                            dev.index, _stream(dev)))
        ctx.save_for_backward(x, weight, mean, invstd)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        x, weight, mean, invstd = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        if not (need_x or need_w or need_b):
            return None, None, None, None, None, None, None
        dy = _aligned(grad_output)
        n, c, h, w = x.shape
        dev = x.device
        if native_reductions(x):
            sum_dy, sum_dy_xmu, gw, gb = (torch.empty(c, dtype=torch.float32, device=dev) for _ in range(4))
            ws, ws_bytes = _workspace(n * h * w, c, dev)
            N.check(N.lib().b2_bn_backward_reduce(dy.data_ptr(), x.data_ptr(), n * h * w, c, N.B2_DT_BFLOAT16, mean.data_ptr(),
                                                  invstd.data_ptr(), sum_dy.data_ptr(), sum_dy_xmu.data_ptr(), gw.data_ptr(),
                                                  gb.data_ptr(), _ptr(ws), ws_bytes, dev.index, _stream(dev)))
        else:
            sum_dy, sum_dy_xmu, gw, gb = torch.batch_norm_backward_reduce(dy, x, mean, invstd, weight, need_x, need_w, need_b)
        dx = _backward_elemt(dy, x, weight, mean, invstd, sum_dy, sum_dy_xmu) if need_x else None
        return dx, gw if need_w else None, gb if need_b else None, None, None, None, None


class _BatchStats(torch.autograd.Function):
    """The first half of a BatchNorm that ``_Normalise`` finishes, for inputs where ``native_reductions`` holds: the batch
    statistics and the running-statistics update.  Returns x itself (autograd hands back an alias), mean, var and an invstd
    that ``_Normalise`` fills.  Its backward is the ``dx`` pass, from the gradient and the sums ``_Normalise.backward``
    left in ``sums``.  Saves what ``_NativeBatchNorm`` saves.

    Two autograd nodes keep the unfused graph's order: a ResNet block creates this one before its downsample branch and
    ``_Normalise`` after it, as the unfused bn3 and residual add are, so backward runs the branches in the same order and
    frees what the unfused step frees when it does."""

    @staticmethod
    def forward(ctx, x, weight, running_mean, running_var, momentum, sums):
        mean, var = _batch_stats(x, running_mean, running_var, momentum)
        invstd = torch.empty(x.shape[1], dtype=torch.float32, device=x.device)
        ctx.save_for_backward(x, weight, mean, invstd)
        ctx.sums = sums
        ctx.mark_non_differentiable(mean, var, invstd)
        return x, mean, var, invstd

    @staticmethod
    @once_differentiable
    def backward(ctx, dy, _mean, _var, _invstd):
        x, weight, mean, invstd = ctx.saved_tensors
        sum_dy, sum_dy_xmu = ctx.sums.pop()
        dx = _backward_elemt(dy, x, weight, mean, invstd, sum_dy, sum_dy_xmu) if ctx.needs_input_grad[0] else None
        return dx, None, None, None, None, None


class _Normalise(torch.autograd.Function):
    """The normalise pass of a BatchNorm whose statistics ``_BatchStats`` took: y = BatchNorm(x), or with ``relu``
    z = ``relu_(y + residual)`` (``relu_(y)`` without a residual) in the same pass, with the bits of the unfused ops
    (DESIGN.md 2.4).  Its backward is the backward reduce, on dy = ``threshold_backward(dz, z, 0)`` formed in the same
    pass with ``relu``; it returns dy (also the residual's gradient) and the weight / bias gradients, and leaves the sums
    to ``_BatchStats.backward``.  Saves z with ``relu``, which the unfused ReLU saved too."""

    @staticmethod
    def forward(ctx, x, residual, weight, bias, mean, var, invstd, eps, relu, sums):
        n, c, h, w = x.shape
        dev = x.device
        y = torch.empty_like(x, memory_format=torch.channels_last)
        if relu:
            N.check(N.lib().b2_bn_forward_relu(x.data_ptr(), _ptr(residual), y.data_ptr(), n * h * w, c, N.B2_DT_BFLOAT16,
                                               weight.data_ptr(), bias.data_ptr(), mean.data_ptr(), var.data_ptr(), float(eps),
                                               invstd.data_ptr(), dev.index, _stream(dev)))
        else:
            N.check(N.lib().b2_bn_forward_elemt(x.data_ptr(), y.data_ptr(), n * h * w, c, N.B2_DT_BFLOAT16, weight.data_ptr(),
                                                bias.data_ptr(), mean.data_ptr(), var.data_ptr(), float(eps), invstd.data_ptr(),
                                                dev.index, _stream(dev)))
        ctx.save_for_backward(x, mean, invstd, y if relu else None)
        ctx.relu, ctx.sums = relu, sums
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        x, mean, invstd, z = ctx.saved_tensors
        c = x.shape[1]
        sum_dy, sum_dy_xmu = (torch.empty(c, dtype=torch.float32, device=x.device) for _ in range(2))
        dy, gw, gb = _normalise_backward(grad_output, x, z, mean, invstd, sum_dy, sum_dy_xmu)
        ctx.sums.append((sum_dy, sum_dy_xmu))
        need_r, need_w, need_b = ctx.needs_input_grad[1:4]
        return dy, dy if need_r else None, gw if need_w else None, gb if need_b else None, None, None, None, None, None, None


def _normalise_backward(grad_output, x, z, mean, invstd, sum_dy, sum_dy_xmu):
    """The backward reduce of a native normalise into sum_dy / sum_dy_xmu: (dy, grad_weight, grad_bias).  With z (the
    output of a normalise that ran the ReLU) dy = threshold_backward(grad_output, z, 0), formed in the same pass."""
    n, c, h, w = x.shape
    dev = x.device
    if z is None:
        dy = _aligned(grad_output)
    elif grad_output.is_contiguous(memory_format=torch.channels_last) and grad_output.data_ptr() % 16 == 0:
        dz, dy = grad_output, torch.empty_like(x, memory_format=torch.channels_last)
    else:
        # a gradient in another layout (a mean's backward hands ResNet's last block an NCHW one) is taken into dy and
        # masked in place: no more activation-sized tensors are alive than in the unfused ReLU's backward
        dz = dy = _aligned(grad_output, copy=True)
    gw, gb = (torch.empty(c, dtype=torch.float32, device=dev) for _ in range(2))
    ws, ws_bytes = _workspace(n * h * w, c, dev)
    if z is not None:
        N.check(N.lib().b2_bn_backward_reduce_relu(dz.data_ptr(), z.data_ptr(), x.data_ptr(), dy.data_ptr(), n * h * w, c,
                                                   N.B2_DT_BFLOAT16, mean.data_ptr(), invstd.data_ptr(), sum_dy.data_ptr(),
                                                   sum_dy_xmu.data_ptr(), gw.data_ptr(), gb.data_ptr(), _ptr(ws), ws_bytes,
                                                   dev.index, _stream(dev)))
    else:
        N.check(N.lib().b2_bn_backward_reduce(dy.data_ptr(), x.data_ptr(), n * h * w, c, N.B2_DT_BFLOAT16, mean.data_ptr(),
                                              invstd.data_ptr(), sum_dy.data_ptr(), sum_dy_xmu.data_ptr(), gw.data_ptr(),
                                              gb.data_ptr(), _ptr(ws), ws_bytes, dev.index, _stream(dev)))
    return dy, gw, gb


# ATen reduces with its channels-last kernels only under 32-bit indexing (canUse32BitIndexMath: fewer than 2^31 - 1
# elements); above that it takes its general path, whose bits the native reductions do not restate.
_INDEX32_LIMIT = 2**31 - 1


def native_reductions(x: torch.Tensor) -> bool:
    """True when the two reductions of an eligible input run natively (``b2_bn_stats`` / ``b2_bn_backward_reduce``): where
    ATen itself would run its channels-last kernels.  Larger inputs keep ATen's own reduction calls."""
    return x.numel() < _INDEX32_LIMIT


def _aligned(t: torch.Tensor, copy: bool = False) -> torch.Tensor:
    """t as the kernels read a gradient: channels-last contiguous and 16-byte aligned (a gradient can be a view that is
    neither), copied only where it is not (always with ``copy``)."""
    if not copy and t.is_contiguous(memory_format=torch.channels_last) and t.data_ptr() % 16 == 0:
        return t
    return t.clone(memory_format=torch.channels_last)


def _ptr(t) -> int:
    return 0 if t is None else t.data_ptr()


def _workspace(rows: int, channels: int, dev: torch.device):
    """Scratch for the reductions' grid_y merge, from torch's caching allocator (stream-ordered), or None."""
    geom, nbytes = (ctypes.c_int * 4)(), ctypes.c_size_t()
    N.check(N.lib().b2_bn_reduce_plan(rows, channels, geom, ctypes.byref(nbytes)))
    if nbytes.value == 0:
        return None, 0
    return torch.empty(nbytes.value // 4, dtype=torch.float32, device=dev), nbytes.value


def native_eligible(bn: nn.BatchNorm2d, x: torch.Tensor) -> bool:
    """True when ``bn(x)`` can run on the native kernels: training with batch statistics, a 4-D CUDA channels-last-
    contiguous bf16 input with channels % 8 == 0, at least 2 values per channel and a 16-byte-aligned data
    pointer, fp32 affine parameters and fp32 running statistics (or none), outside ``torch.compile`` tracing."""
    if not bn.training or torch.compiler.is_compiling():
        return False
    if x.dim() != 4 or not x.is_cuda or x.dtype != torch.bfloat16 or not x.is_contiguous(memory_format=torch.channels_last):
        return False
    n, c, h, w = x.shape
    if c != bn.num_features or c % 8 != 0 or n * h * w < 2 or x.data_ptr() % 16 != 0:
        return False
    if not bn.affine or bn.weight.dtype != torch.float32 or bn.bias.dtype != torch.float32:
        return False
    if bn.weight.device != x.device or bn.bias.device != x.device:
        return False
    if bn.track_running_stats:
        for t in (bn.running_mean, bn.running_var):
            if t is None or t.dtype != torch.float32 or t.device != x.device or not t.is_contiguous():
                return False
    return bn.weight.is_contiguous() and bn.bias.is_contiguous()


class BatchNorm2d(nn.BatchNorm2d):
    """``nn.BatchNorm2d`` whose training elementwise passes run on native kernels where ``native_eligible`` holds."""

    def forward(self, input: torch.Tensor) -> torch.Tensor:  # noqa: A002
        if not native_eligible(self, input):
            return super().forward(input)
        return _NativeBatchNorm.apply(input, self.weight, self.bias, *self._training_step(), self.eps)

    def batch_stats(self, input: torch.Tensor):  # noqa: A002
        """The first half of ``self(input)`` on the native kernels, for an input where ``native_eligible`` and
        ``native_reductions`` hold: the batch statistics and the running-statistics update.  ``normalise`` takes the
        result and finishes the layer; ``torchx_b200.nn.resnet`` runs a block's residual branch between the two."""
        running_mean, running_var, momentum = self._training_step()
        sums = []  # the backward reduce's sums, from _Normalise.backward to _BatchStats.backward
        return _BatchStats.apply(input, self.weight, running_mean, running_var, momentum, sums) + (sums,)

    def normalise(self, stats, residual: Optional[torch.Tensor] = None, relu: bool = False) -> torch.Tensor:
        """The rest of ``self(input)`` from ``batch_stats(input)``: the BatchNorm output, or with ``relu``
        ``relu_(output + residual)`` (``relu_(output)`` without a residual) in the same pass, with the same bits.  A
        residual must be a bf16 channels-last tensor of the input's shape and device, 16-byte aligned."""
        x, mean, var, invstd, sums = stats
        return _Normalise.apply(x, residual, self.weight, self.bias, mean, var, invstd, self.eps, relu, sums)

    def _training_step(self):
        """nn.BatchNorm2d.forward's preamble in training mode: (running_mean, running_var, exponential_average_factor)."""
        exponential_average_factor = 0.0 if self.momentum is None else self.momentum
        if self.track_running_stats and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
            if self.momentum is None:  # cumulative moving average
                exponential_average_factor = 1.0 / float(self.num_batches_tracked)
            else:
                exponential_average_factor = self.momentum
        running_mean = self.running_mean if self.track_running_stats else None
        running_var = self.running_var if self.track_running_stats else None
        return running_mean, running_var, exponential_average_factor


def convert_batchnorm(module: nn.Module) -> nn.Module:
    """Switch every layer of ``module`` whose type is exactly ``nn.BatchNorm2d`` to ``BatchNorm2d``, in place (its
    ``__class__`` changes; parameters, buffers, hooks and state-dict keys stay the same objects).  Subclasses,
    ``SyncBatchNorm`` and ``BatchNorm1d`` / ``BatchNorm3d`` are left alone.  Returns ``module``."""
    for m in module.modules():
        if type(m) is nn.BatchNorm2d:
            m.__class__ = BatchNorm2d
    return module
