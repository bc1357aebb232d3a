"""Native BatchNorm2d, the parts that need no GPU: the C ABI entries and every argument check, which inputs take the native
path, the converted module on CPU tensors (where it is nn.BatchNorm2d, bit for bit), and what the conversion touches."""
import copy
import ctypes
import os
import pickle
import re

import pytest
import torch
from torch import nn

from torchx_b200.ddp import _native as N
from torchx_b200.nn import BatchNorm2d, SyncBatchNorm, convert_batchnorm, native_eligible

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- C ABI -------------------------------------------------------------------------------------------------------------
def test_header_declares_the_entry_points_and_the_binding_resolves_them():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    assert re.search(r"int b2_bn_forward_elemt\(const void\* x, void\* y, size_t rows, size_t channels, int dtype, const float\* weight,", src)
    assert re.search(r"int b2_bn_backward_elemt\(const void\* dy, const void\* x, void\* dx, size_t rows, size_t channels, int dtype,", src)
    assert int(re.search(r"#define\s+B2_ABI_VERSION\s+(\d+)", src).group(1)) == N.B2_ABI_VERSION == 3
    L = N.lib()
    for name, nargs in (("b2_bn_forward_elemt", 13), ("b2_bn_backward_elemt", 13)):
        assert name in N.SYMBOLS
        assert getattr(L, name).restype is ctypes.c_int and len(getattr(L, name).argtypes) == nargs


def _err():
    return N.lib().b2_last_error().decode()


P = 1 << 20  # an aligned fake device address: every call below fails validation before anything touches it


def _fwd(x=P, y=P, rows=64, channels=16, dtype=N.B2_DT_BFLOAT16, weight=P, bias=P, mean=P, var=P, invstd=P):
    return N.lib().b2_bn_forward_elemt(x, y, rows, channels, dtype, weight, bias, mean, var, 1e-5, invstd, 0, None)


def _bwd(dy=P, x=P, dx=P, rows=64, channels=16, dtype=N.B2_DT_BFLOAT16, weight=P, mean=P, invstd=P, sum_dy=P, sum_dy_xmu=P):
    return N.lib().b2_bn_backward_elemt(dy, x, dx, rows, channels, dtype, weight, mean, invstd, sum_dy, sum_dy_xmu, 0, None)


@pytest.mark.parametrize("call,fn", [(_fwd, "b2_bn_forward_elemt"), (_bwd, "b2_bn_backward_elemt")])
def test_validation_messages(call, fn):
    for dtype in (N.B2_DT_FLOAT16, N.B2_DT_FLOAT32, N.B2_DT_INT32, 7):
        assert call(dtype=dtype) == N.B2_EINVAL
        assert f"{fn}: dtype {dtype} is not B2_DT_BFLOAT16" in _err()
    for c in (0, 12, 20):
        assert call(channels=c) == N.B2_EINVAL
        assert f"{fn}: channels={c} must be a positive multiple of 8" in _err()
    for rows in (0, 1):
        assert call(rows=rows) == N.B2_EINVAL
        assert f"{fn}: rows={rows}, batch statistics need at least 2" in _err()
    assert call(x=None) == N.B2_EINVAL
    assert f"{fn}: null x" in _err()
    assert call(x=P + 8) == N.B2_EINVAL
    assert f"{fn}: x is not 16-byte aligned" in _err()
    assert call(weight=None) == N.B2_EINVAL
    assert f"{fn}: null weight" in _err()
    assert call(weight=P + 2) == N.B2_EINVAL
    assert f"{fn}: weight is not 4-byte aligned" in _err()
    assert call(mean=None) == N.B2_EINVAL
    assert f"{fn}: null mean" in _err()
    assert call(invstd=P + 1) == N.B2_EINVAL
    assert "invstd is not 4-byte aligned" in _err()


def test_validation_of_the_pass_specific_pointers():
    assert _fwd(y=P + 8) == N.B2_EINVAL and "b2_bn_forward_elemt: y is not 16-byte aligned" in _err()
    assert _fwd(bias=None) == N.B2_EINVAL and "b2_bn_forward_elemt: null bias" in _err()
    assert _fwd(var=P + 1) == N.B2_EINVAL and "b2_bn_forward_elemt: var is not 4-byte aligned" in _err()
    assert _fwd(invstd=None) == N.B2_EINVAL and "b2_bn_forward_elemt: null save_invstd" in _err()
    assert _bwd(dy=None) == N.B2_EINVAL and "b2_bn_backward_elemt: null dy" in _err()
    assert _bwd(dx=None) == N.B2_EINVAL and "b2_bn_backward_elemt: null dx" in _err()
    assert _bwd(dx=P + 8) == N.B2_EINVAL and "b2_bn_backward_elemt: dx is not 16-byte aligned" in _err()
    assert _bwd(sum_dy=None) == N.B2_EINVAL and "b2_bn_backward_elemt: null sum_dy" in _err()
    assert _bwd(sum_dy_xmu=P + 2) == N.B2_EINVAL and "b2_bn_backward_elemt: sum_dy_xmu is not 4-byte aligned" in _err()


# ---- which inputs take the native path ----------------------------------------------------------------------------------
class _FakeCuda:
    """Just enough of a tensor for native_eligible, so the predicate can be checked case by case without a GPU."""

    def __init__(self, shape=(4, 16, 5, 5), dtype=torch.bfloat16, cl=True, ptr=1 << 20, is_cuda=True, device=None):
        self.shape, self.dtype, self._cl, self._ptr, self.is_cuda = shape, dtype, cl, ptr, is_cuda
        self.device = device

    def dim(self):
        return len(self.shape)

    def is_contiguous(self, memory_format=torch.contiguous_format):
        return self._cl if memory_format == torch.channels_last else not self._cl

    def data_ptr(self):
        return self._ptr


def _bn(c=16, **kw):
    bn = BatchNorm2d(c, **kw)
    bn.train()
    return bn


def _x(bn, **kw):
    return _FakeCuda(device=bn.weight.device if bn.weight is not None else torch.device("cpu"), **kw)


def test_eligibility_case_by_case():
    bn = _bn()
    assert native_eligible(bn, _x(bn))
    assert not native_eligible(bn, _x(bn, dtype=torch.float16))  # torch runs cuDNN's BatchNorm there
    assert not native_eligible(bn, _x(bn, dtype=torch.float32))
    assert not native_eligible(bn, _x(bn, cl=False))
    assert not native_eligible(bn, _x(bn, is_cuda=False))
    assert not native_eligible(bn, _x(bn, shape=(4, 16, 25)))
    assert not native_eligible(bn, _x(bn, ptr=(1 << 20) + 8))
    assert not native_eligible(bn, _x(bn, shape=(1, 16, 1, 1)))  # one value per channel
    assert native_eligible(bn, _x(bn, shape=(2, 16, 1, 1)))
    bn12 = _bn(12)
    assert not native_eligible(bn12, _x(bn12, shape=(4, 12, 5, 5)))
    assert not native_eligible(bn, _x(bn, shape=(4, 24, 5, 5)))  # channels differ from num_features: torch's error
    bn.eval()
    assert not native_eligible(bn, _x(bn))
    assert not native_eligible(_bn(affine=False), _x(_bn()))
    half = _bn()
    half.half()
    assert not native_eligible(half, _x(half))  # fp16 parameters
    rs = _bn()
    rs.running_var = rs.running_var.double()
    assert not native_eligible(rs, _x(rs))
    assert native_eligible(_bn(track_running_stats=False), _x(bn))
    bn.train()
    compiling = torch.compiler.is_compiling
    try:
        torch.compiler.is_compiling = lambda: True
        assert not native_eligible(bn, _x(bn))
    finally:
        torch.compiler.is_compiling = compiling


# ---- the module on CPU tensors is nn.BatchNorm2d -------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, {"momentum": None}, {"track_running_stats": False}, {"affine": False}])
def test_converted_module_is_bit_equal_on_cpu(kw):
    torch.manual_seed(0)
    ref = nn.BatchNorm2d(16, **kw)
    if ref.affine:
        with torch.no_grad():
            ref.weight.uniform_(0.5, 1.5)
            ref.bias.uniform_(-0.5, 0.5)
    mine = copy.deepcopy(ref)
    convert_batchnorm(mine)
    assert type(mine) is BatchNorm2d
    for step in range(3):
        x = torch.randn(4, 16, 5, 5).contiguous(memory_format=torch.channels_last) * (step + 1) + step
        xr, xm = x.clone().requires_grad_(), x.clone().requires_grad_()
        yr, ym = ref(xr), mine(xm)
        assert torch.equal(yr, ym)
        yr.square().sum().backward()
        ym.square().sum().backward()
        assert torch.equal(xr.grad, xm.grad)
    for (n, a), (_, b) in zip(ref.state_dict().items(), mine.state_dict().items()):
        assert torch.equal(a, b), n
    ref.eval()
    mine.eval()
    x = torch.randn(2, 16, 3, 3)
    assert torch.equal(ref(x), mine(x))


def test_torch_errors_are_unchanged():
    bn = convert_batchnorm(nn.BatchNorm2d(8))
    with pytest.raises(ValueError, match="expected 4D input"):
        bn(torch.randn(4, 8))
    with pytest.raises(ValueError, match="Expected more than 1 value per channel"):
        bn(torch.randn(1, 8, 1, 1))


# ---- the conversion -----------------------------------------------------------------------------------------------------
class _MyBN(nn.BatchNorm2d):
    pass


def test_conversion_touches_only_exact_batchnorm2d_and_keeps_identity():
    net = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), _MyBN(8), nn.BatchNorm1d(8), nn.BatchNorm3d(8), nn.SyncBatchNorm(8),
                        SyncBatchNorm(8), nn.Sequential(nn.BatchNorm2d(16)))
    calls = []
    h = net[1].register_forward_hook(lambda *a: calls.append(1))
    params = {n: p for n, p in net.named_parameters()}
    bufs = {n: b for n, b in net.named_buffers()}
    keys = list(net.state_dict())
    assert convert_batchnorm(net) is net
    assert [type(m) for m in net] == [nn.Conv2d, BatchNorm2d, _MyBN, nn.BatchNorm1d, nn.BatchNorm3d, nn.SyncBatchNorm, SyncBatchNorm,
                                      nn.Sequential]
    assert type(net[7][0]) is BatchNorm2d
    assert isinstance(net[1], nn.BatchNorm2d)
    assert all(p is params[n] for n, p in net.named_parameters())
    assert all(b is bufs[n] for n, b in net.named_buffers())
    assert list(net.state_dict()) == keys
    net[1].eval()
    net[1](torch.randn(2, 8, 3, 3))
    assert calls == [1]
    h.remove()
    convert_batchnorm(net)  # idempotent
    assert type(net[1]) is BatchNorm2d


def test_converted_module_survives_deepcopy_and_pickle():
    net = convert_batchnorm(nn.Sequential(nn.BatchNorm2d(8)))
    with torch.no_grad():
        net[0].running_mean.fill_(0.25)
    for other in (copy.deepcopy(net), pickle.loads(pickle.dumps(net))):
        assert type(other[0]) is BatchNorm2d
        for (n, a), (_, b) in zip(net.state_dict().items(), other.state_dict().items()):
            assert torch.equal(a, b), n
