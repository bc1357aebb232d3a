"""ReLU and the residual add inside the native BatchNorm passes, the parts that need no GPU: the fused C entry points and
their argument checks, what ``fuse_resnet`` swaps and keeps, and when a block takes its fused forward."""
import copy
import ctypes
import os
import pickle
import re

import pytest
import torch
from torch import nn

from torchx_b200.ddp import _native as N
from torchx_b200.nn import BatchNorm2d, SyncBatchNorm, convert_batchnorm, fuse_resnet
from torchx_b200.nn import resnet as R

torchvision = pytest.importorskip("torchvision")
from torchvision.models import resnet as tv  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- C ABI -------------------------------------------------------------------------------------------------------------
def test_header_declares_the_fused_entry_points():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    assert re.search(r"int b2_bn_forward_relu\(const void\* x, const void\* residual, void\* y, size_t rows, size_t channels,", src)
    assert re.search(r"int b2_bn_backward_reduce_relu\(const void\* dz, const void\* z, const void\* x, void\* dy, size_t rows,", src)
    assert int(re.search(r"#define\s+B2_ABI_VERSION\s+(\d+)", src).group(1)) == N.B2_ABI_VERSION == 3
    L = N.lib()
    for name, nargs in (("b2_bn_forward_relu", 14), ("b2_bn_backward_reduce_relu", 17)):
        assert name in N.SYMBOLS
        assert getattr(L, name).restype is ctypes.c_int and len(getattr(L, name).argtypes) == nargs


def _err():
    return N.lib().b2_last_error().decode()


P = 1 << 20  # an aligned fake device address: every call below fails validation before anything touches it


def _fwd(x=P, residual=P, y=P, rows=64, channels=16, dtype=N.B2_DT_BFLOAT16, weight=P, bias=P, mean=P, var=P, invstd=P):
    return N.lib().b2_bn_forward_relu(x, residual, y, rows, channels, dtype, weight, bias, mean, var, 1e-5, invstd, 0, None)


def _reduce(dz=P, z=P, x=P, dy=P, rows=64, channels=16, dtype=N.B2_DT_BFLOAT16, mean=P, invstd=P, sum_dy=P, sum_dy_xmu=P, gw=P, gb=P,
            ws=None, ws_bytes=0):
    return N.lib().b2_bn_backward_reduce_relu(dz, z, x, dy, rows, channels, dtype, mean, invstd, sum_dy, sum_dy_xmu, gw, gb, ws, ws_bytes,
                                              0, None)


@pytest.mark.parametrize("call,fn", [(_fwd, "b2_bn_forward_relu"), (_reduce, "b2_bn_backward_reduce_relu")])
def test_validation_messages(call, fn):
    assert call(dtype=N.B2_DT_FLOAT16) == N.B2_EINVAL and f"{fn}: dtype {N.B2_DT_FLOAT16} is not B2_DT_BFLOAT16" in _err()
    assert call(channels=12) == N.B2_EINVAL and f"{fn}: channels=12 must be a positive multiple of 8" in _err()
    assert call(rows=1) == N.B2_EINVAL and f"{fn}: rows=1, batch statistics need at least 2" in _err()
    assert call(x=None) == N.B2_EINVAL and f"{fn}: null x" in _err()
    assert call(x=P + 8) == N.B2_EINVAL and f"{fn}: x is not 16-byte aligned" in _err()
    assert call(mean=None) == N.B2_EINVAL and f"{fn}: null mean" in _err()
    assert call(invstd=P + 2) == N.B2_EINVAL and "invstd is not 4-byte aligned" in _err()


def test_validation_of_the_fused_pointers():
    assert _fwd(residual=P + 8) == N.B2_EINVAL and "b2_bn_forward_relu: residual is not 16-byte aligned" in _err()
    assert _fwd(y=None) == N.B2_EINVAL and "b2_bn_forward_relu: null y" in _err()
    assert _fwd(bias=P + 1) == N.B2_EINVAL and "b2_bn_forward_relu: bias is not 4-byte aligned" in _err()
    # a null residual is no residual: the call gets as far as the next check
    assert _fwd(residual=None, var=None) == N.B2_EINVAL and "b2_bn_forward_relu: null var" in _err()
    for name in ("dz", "z", "dy"):
        assert _reduce(**{name: None}) == N.B2_EINVAL and f"b2_bn_backward_reduce_relu: null {name}" in _err()
        assert _reduce(**{name: P + 4}) == N.B2_EINVAL and f"b2_bn_backward_reduce_relu: {name} is not 16-byte aligned" in _err()
    assert _reduce(rows=268435456, channels=8) == N.B2_EINVAL
    assert "b2_bn_backward_reduce_relu: rows*channels=268435456 x 8 must be below 2^31 - 1 elements" in _err()
    assert _reduce(gb=None) == N.B2_EINVAL and "b2_bn_backward_reduce_relu: null grad_bias" in _err()
    assert _reduce(rows=2560, channels=64) == N.B2_EINVAL and "b2_bn_backward_reduce_relu: null workspace" in _err()


# ---- fuse_resnet --------------------------------------------------------------------------------------------------------
def _models():
    torch.manual_seed(0)
    return [tv.resnet18(), tv.resnet50()]


def test_swaps_exactly_the_resnet_types():
    for m in _models():
        before = {n: type(x) for n, x in m.named_modules()}
        assert fuse_resnet(m) is m
        for n, x in m.named_modules():
            old = before[n]
            if old in (tv.Bottleneck, tv.BasicBlock, tv.ResNet):
                assert type(x) is getattr(R, "Fused" + old.__name__) and isinstance(x, old), n
                assert type(x).__module__ == R.__name__ and type(x).__qualname__ == "Fused" + old.__name__
            else:
                assert type(x) is old, n


def test_leaves_subclasses_and_other_models_alone():
    class MyBlock(tv.BasicBlock):
        pass

    seq = nn.Sequential(MyBlock(8, 8), nn.Conv2d(8, 8, 1), nn.BatchNorm2d(8), nn.ReLU())
    fuse_resnet(seq)
    assert [type(x) for x in seq] == [MyBlock, nn.Conv2d, nn.BatchNorm2d, nn.ReLU]


def test_keeps_parameters_buffers_keys_and_hooks():
    m = convert_batchnorm(_models()[1])
    params = [id(p) for p in m.parameters()]
    buffers = [id(b) for b in m.buffers()]
    keys = list(m.state_dict())
    h = m.layer1[0].register_forward_hook(lambda *a: None)
    fuse_resnet(m)
    assert [id(p) for p in m.parameters()] == params and [id(b) for b in m.buffers()] == buffers
    assert list(m.state_dict()) == keys
    assert h.id in m.layer1[0]._forward_hooks
    assert all(type(b) is BatchNorm2d for b in m.modules() if isinstance(b, nn.BatchNorm2d))


def test_idempotent_and_survives_deepcopy_and_pickle():
    m = fuse_resnet(convert_batchnorm(_models()[0]))
    types = [type(x) for x in m.modules()]
    fuse_resnet(m)
    assert [type(x) for x in m.modules()] == types
    for twin in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        assert [type(x) for x in twin.modules()] == types
        assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), twin.state_dict().values()))


def test_without_torchvision_does_nothing(monkeypatch):
    import builtins

    real = builtins.__import__

    def no_torchvision(name, *a, **kw):
        if name.startswith("torchvision"):
            raise ImportError(name)
        return real(name, *a, **kw)

    monkeypatch.setattr(builtins, "__import__", no_torchvision)
    m = tv.resnet18()
    fuse_resnet(m)
    assert type(m) is tv.ResNet and type(m.layer1[0]) is tv.BasicBlock


# ---- when a block fuses ---------------------------------------------------------------------------------------------------
def _block():
    blk = convert_batchnorm(tv.Bottleneck(64, 16))
    fuse_resnet(blk)
    return blk


def _bns(blk):
    return (blk.bn1, blk.bn2, blk.bn3)


def test_fusable_conditions():
    blk = _block()
    assert R._fusable(blk, _bns(blk))
    blk.eval()
    assert not R._fusable(blk, _bns(blk))
    blk.train()
    h = blk.bn2.register_forward_pre_hook(lambda *a: None)
    assert not R._fusable(blk, _bns(blk))
    h.remove()
    h = blk.relu.register_forward_hook(lambda *a: None)
    assert not R._fusable(blk, _bns(blk))
    h.remove()
    h = blk.bn3.register_full_backward_hook(lambda *a: None)
    assert not R._fusable(blk, _bns(blk))
    h.remove()
    h = nn.modules.module.register_module_forward_hook(lambda *a: None)
    assert not R._fusable(blk, _bns(blk))
    h.remove()
    assert R._fusable(blk, _bns(blk))
    for bad in (nn.BatchNorm2d(64), SyncBatchNorm(64)):
        assert not R._fusable(blk, (blk.bn1, blk.bn2, bad))
    blk.relu = nn.ReLU6()
    assert not R._fusable(blk, _bns(blk))


def test_residual_conditions():
    x = torch.empty(2, 16, 3, 3, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    assert R._residual_ok(torch.empty_like(x), x)
    assert not R._residual_ok(torch.empty_like(x, dtype=torch.float16), x)
    assert not R._residual_ok(torch.empty_like(x, dtype=torch.float32), x)
    assert not R._residual_ok(torch.empty(2, 16, 3, 3, dtype=torch.bfloat16), x)  # NCHW
    assert not R._residual_ok(torch.empty(2, 16, 3, 4, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last), x)
    flat = torch.empty(2 * 16 * 9 + 1, dtype=torch.bfloat16)
    odd = flat[1:].view(2, 3, 3, 16).permute(0, 3, 1, 2)  # channels-last view at a 2-byte offset
    assert odd.is_contiguous(memory_format=torch.channels_last) and not R._residual_ok(odd, x)


@pytest.mark.parametrize("train", [True, False])
def test_cpu_forward_and_backward_are_the_unfused_bits(train):
    """On CPU tensors every layer refuses the native path: the fused forward must run the unfused ops."""
    torch.manual_seed(1)
    for base in (tv.resnet18(), tv.Bottleneck(64, 16, downsample=nn.Sequential(nn.Conv2d(64, 64, 1), nn.BatchNorm2d(64)))):
        plain = convert_batchnorm(copy.deepcopy(base))
        fused = fuse_resnet(convert_batchnorm(copy.deepcopy(base)))
        plain.train(train)
        fused.train(train)
        x = torch.randn(2, 3 if isinstance(base, tv.ResNet) else 64, 32, 32)
        a, b = plain(x.clone().requires_grad_()), fused(x.clone().requires_grad_())
        assert torch.equal(a, b)
        a.sum().backward()
        b.sum().backward()
        for (n, p), q in zip(plain.named_parameters(), fused.parameters()):
            assert torch.equal(p.grad, q.grad), n
        for (n, p), q in zip(plain.named_buffers(), fused.buffers()):
            assert torch.equal(p, q), n

