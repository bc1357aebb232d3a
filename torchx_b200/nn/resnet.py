"""torchvision's ResNet blocks with each BatchNorm's ReLU, and the residual add before the last one, inside the native
BatchNorm passes (``BatchNorm2d.batch_stats`` / ``normalise``, DESIGN.md 2.5).

``fuse_resnet`` switches the ``__class__`` of every module whose type is exactly ``torchvision.models.resnet.Bottleneck``,
``BasicBlock`` or ``ResNet`` to a subclass whose forward runs

* ``Bottleneck``: bn1 + ReLU, bn2 + ReLU, bn3 + residual + ReLU;
* ``BasicBlock``: bn1 + ReLU, bn2 + residual + ReLU;
* ``ResNet``: the stem's bn1 + ReLU.

Each is the unfused forward's result bit for bit.  A block takes its parent's forward unchanged unless it is training,
its BatchNorms are exactly ``torchx_b200.nn.BatchNorm2d`` or exactly ``torchx_b200.nn.SyncBatchNorm`` on the fabric
(``SyncBatchNorm._fusable``), its ReLU is exactly ``nn.ReLU``, no hook is registered on those layers and no global module
hook exists, and it is not traced by ``torch.compile``.  Within a fused forward, a ``BatchNorm2d`` (or a SyncBatchNorm at
one rank) whose input ``native_eligible`` / ``native_reductions`` refuses runs the unfused ``relu(bn(x) [+ residual])``, and a
layer whose residual is not a bf16 channels-last tensor of the output's shape adds it and runs the ReLU after its
normalise.  A SyncBatchNorm over several ranks always runs as ``batch_stats`` / ``normalise``, on ATen's
compute where its input is not eligible: whether it fuses is decided from nothing but the block, which is the same on
every rank, so every rank issues the block's exchanges and allreduces in the same order (DESIGN.md 2.5).  So fp16 and fp32
activations and eval mode compute exactly what they computed before.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch
from torch import nn
from torch.nn.modules import module as _module

from torchx_b200.nn.batchnorm import SyncBatchNorm
from torchx_b200.nn.bn2d import BatchNorm2d, native_eligible, native_reductions


def _hooked(m: nn.Module) -> bool:
    return bool(m._forward_hooks or m._forward_pre_hooks or m._backward_hooks or m._backward_pre_hooks)


def _fusable(block: nn.Module, bns) -> bool:
    """The conditions a block checks before it takes its fused forward (the module docstring)."""
    if not block.training or torch.compiler.is_compiling():
        return False
    if type(block.relu) is not nn.ReLU or _hooked(block.relu):
        return False
    if any(_hooked(bn) or not (type(bn) is BatchNorm2d or (type(bn) is SyncBatchNorm and bn._fusable())) for bn in bns):
        return False
    return not (_module._global_forward_hooks or _module._global_forward_pre_hooks or _module._global_backward_hooks
                or _module._global_backward_pre_hooks)


def _two_phase(bn: nn.Module, x: torch.Tensor) -> bool:
    """Whether ``bn`` runs as ``batch_stats`` / ``normalise``: always for a SyncBatchNorm over several ranks (its collectives
    must not depend on this rank's input), otherwise where the native kernels cover x."""
    if type(bn) is SyncBatchNorm and bn._comm().world > 1:
        return True
    return native_eligible(bn, x) and native_reductions(x)


def _bn_relu(bn: nn.Module, relu: nn.ReLU, x: torch.Tensor, residual: Optional[Callable[[], torch.Tensor]] = None) -> torch.Tensor:
    """``relu(bn(x) + residual())`` (``relu(bn(x))`` without a residual), fused where the kernels cover the inputs.  The
    residual branch runs after the BatchNorm's statistics and before its normalise, so that the autograd graph keeps the
    unfused forward's node order (``_BatchStats``)."""
    if not _two_phase(bn, x):
        out = bn(x)
        if residual is not None:
            out += residual()
        return relu(out)
    stats = bn.batch_stats(x)
    r = residual() if residual is not None else None
    if r is not None and not _residual_ok(r, x):
        out = bn.normalise(stats)
        out += r
        return relu(out)
    return bn.normalise(stats, r, relu=True)


def _residual_ok(r: torch.Tensor, x: torch.Tensor) -> bool:
    return (r.dtype == torch.bfloat16 and r.device == x.device and r.shape == x.shape
            and r.is_contiguous(memory_format=torch.channels_last) and r.data_ptr() % 16 == 0)


class _FusedBottleneck:
    _fused_bns = ("bn1", "bn2", "bn3")  # the BatchNorms followed by a ReLU; the last one's adds the residual
    _residual_bn = "bn3"

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not _fusable(self, (self.bn1, self.bn2, self.bn3)):
            return super().forward(x)
        out = _bn_relu(self.bn1, self.relu, self.conv1(x))
        out = _bn_relu(self.bn2, self.relu, self.conv2(out))
        return _bn_relu(self.bn3, self.relu, self.conv3(out), lambda: x if self.downsample is None else self.downsample(x))


class _FusedBasicBlock:
    _fused_bns = ("bn1", "bn2")
    _residual_bn = "bn2"

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not _fusable(self, (self.bn1, self.bn2)):
            return super().forward(x)
        out = _bn_relu(self.bn1, self.relu, self.conv1(x))
        return _bn_relu(self.bn2, self.relu, self.conv2(out), lambda: x if self.downsample is None else self.downsample(x))


class _FusedResNet:
    _fused_bns = ("bn1",)
    _residual_bn = None

    def _forward_impl(self, x: torch.Tensor) -> torch.Tensor:
        if not _fusable(self, (self.bn1,)):
            return super()._forward_impl(x)
        x = _bn_relu(self.bn1, self.relu, self.conv1(x))
        x = self.maxpool(x)
        x = self.layer1(x)
        x = self.layer2(x)
        x = self.layer3(x)
        x = self.layer4(x)
        x = self.avgpool(x)
        x = torch.flatten(x, 1)
        return self.fc(x)


_MIXINS = {"FusedBottleneck": ("Bottleneck", _FusedBottleneck), "FusedBasicBlock": ("BasicBlock", _FusedBasicBlock),
           "FusedResNet": ("ResNet", _FusedResNet)}
_classes: Dict[str, type] = {}


def _fused_classes() -> Dict[type, type]:
    """{torchvision class: its fused subclass}, built on first use (torchvision is optional), or {} without torchvision."""
    try:
        from torchvision.models import resnet as tv
    except ImportError:
        return {}
    if not _classes:
        for name, (base, mixin) in _MIXINS.items():
            _classes[name] = type(name, (mixin, getattr(tv, base)), {"__module__": __name__, "__qualname__": name})
    return {getattr(tv, base): _classes[name] for name, (base, _) in _MIXINS.items()}


def __getattr__(name: str) -> type:
    # the fused classes by name, as pickle looks them up
    if name in _MIXINS and _fused_classes():
        return _classes[name]
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")


def fuse_resnet(module: nn.Module) -> nn.Module:
    """Switch every module of ``module`` whose type is exactly torchvision's ``Bottleneck``, ``BasicBlock`` or ``ResNet`` to
    its fused subclass, in place (its ``__class__`` changes; parameters, buffers, hooks and state-dict keys stay the same
    objects, and ``isinstance`` still holds).  Idempotent; without torchvision it does nothing.  Returns ``module``."""
    fused = _fused_classes()
    if fused:
        for m in module.modules():
            cls = fused.get(type(m))
            if cls is not None:
                m.__class__ = cls
    return module
