"""SyncBatchNorm on the native BatchNorm2d kernels, the parts that need no GPU: the three entry points' argument checks,
which inputs take the native path and which keep ATen's compute, and which ResNet blocks fuse with SyncBatchNorm layers."""
import ctypes
import re

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import torchx_b200.distributed as D
import torchx_b200.nn.batchnorm as B
import torchx_b200.nn.resnet as R
from torchx_b200.ddp import _native as N
from torchx_b200.nn import BatchNorm2d, SyncBatchNorm

P = 1 << 20  # an aligned fake device address: every call below fails validation before anything touches it


def _err():
    return N.lib().b2_last_error().decode()


def test_header_declares_the_entry_points_and_the_binding_resolves_them():
    src = open(N.os.path.join(N.INCLUDE_DIR, "b200ddp.h")).read()
    L = N.lib()
    for name, nargs in (("b2_bn_stats_invstd", 11), ("b2_bn_forward_invstd", 13), ("b2_bn_backward_elemt_counts", 15)):
        assert re.search(rf"int {name}\(", src), name
        assert getattr(L, name).restype is ctypes.c_int and len(getattr(L, name).argtypes) == nargs


def _stats(x=P, rows=64, channels=16, dtype=N.B2_DT_BFLOAT16, mean=P, invstd=P, ws=None, ws_bytes=0):
    return N.lib().b2_bn_stats_invstd(x, rows, channels, dtype, mean, invstd, 1e-5, ws, ws_bytes, 0, None)


def _fwd(x=P, residual=None, y=P, relu=0, rows=64, channels=16, dtype=N.B2_DT_BFLOAT16, weight=P, bias=P, mean=P, invstd=P):
    return N.lib().b2_bn_forward_invstd(x, residual, y, relu, rows, channels, dtype, weight, bias, mean, invstd, 0, None)


def _bwd(dy=P, x=P, dx=P, rows=64, channels=16, dtype=N.B2_DT_BFLOAT16, weight=P, mean=P, invstd=P, sum_dy=P, sum_dy_xmu=P,
         counts=P, n_counts=2):
    return N.lib().b2_bn_backward_elemt_counts(dy, x, dx, rows, channels, dtype, weight, mean, invstd, sum_dy, sum_dy_xmu, counts,
                                               n_counts, 0, None)


@pytest.mark.parametrize("call,fn", [(_stats, "b2_bn_stats_invstd"), (_fwd, "b2_bn_forward_invstd"),
                                     (_bwd, "b2_bn_backward_elemt_counts")])
def test_shared_validation(call, fn):
    for dtype in (N.B2_DT_FLOAT16, N.B2_DT_FLOAT32, 7):
        assert call(dtype=dtype) == N.B2_EINVAL and f"{fn}: dtype {dtype} is not B2_DT_BFLOAT16" in _err()
    for c in (0, 12):
        assert call(channels=c) == N.B2_EINVAL and f"{fn}: channels={c} must be a positive multiple of 8" in _err()
    for rows in (0, 1):
        assert call(rows=rows) == N.B2_EINVAL and f"{fn}: rows={rows}, batch statistics need at least 2" in _err()
    assert call(x=None) == N.B2_EINVAL and f"{fn}: null x" in _err()
    assert call(x=P + 8) == N.B2_EINVAL and f"{fn}: x is not 16-byte aligned" in _err()
    assert call(mean=None) == N.B2_EINVAL and f"{fn}: null mean" in _err()
    assert call(invstd=None) == N.B2_EINVAL and f"{fn}: null invstd" in _err()
    assert call(invstd=P + 1) == N.B2_EINVAL and f"{fn}: invstd is not 4-byte aligned" in _err()


def test_statistics_checks():
    assert _stats(rows=1 << 28, channels=16) == N.B2_EINVAL and "must be below 2^31 - 1 elements" in _err()
    geom, nbytes = (ctypes.c_int * 4)(), ctypes.c_size_t()
    assert N.lib().b2_bn_reduce_plan(802816, 64, geom, ctypes.byref(nbytes)) == N.B2_OK and nbytes.value > 0
    assert _stats(rows=802816, channels=64) == N.B2_EINVAL and "b2_bn_stats_invstd: null workspace" in _err()
    assert _stats(rows=802816, channels=64, ws=P, ws_bytes=nbytes.value - 4) == N.B2_EINVAL and "needed" in _err()


def test_forward_checks():
    fn = "b2_bn_forward_invstd"
    assert _fwd(y=P + 8) == N.B2_EINVAL and f"{fn}: y is not 16-byte aligned" in _err()
    assert _fwd(weight=None) == N.B2_EINVAL and f"{fn}: null weight" in _err()
    assert _fwd(bias=P + 2) == N.B2_EINVAL and f"{fn}: bias is not 4-byte aligned" in _err()
    assert _fwd(residual=P + 8, relu=1) == N.B2_EINVAL and f"{fn}: residual is not 16-byte aligned" in _err()


def test_backward_counts_checks():
    fn = "b2_bn_backward_elemt_counts"
    assert _bwd(counts=None) == N.B2_EINVAL and f"{fn}: null counts" in _err()
    assert _bwd(counts=P + 2) == N.B2_EINVAL and f"{fn}: counts is not 4-byte aligned" in _err()
    for n in (0, -1, N.B2_MAX_WORLD + 1):
        assert _bwd(n_counts=n) == N.B2_EINVAL and f"{fn}: n_counts={n} must be in 1..{N.B2_MAX_WORLD}" in _err()
    assert _bwd(dx=None) == N.B2_EINVAL and f"{fn}: null dx" in _err()
    assert _bwd(sum_dy_xmu=P + 2) == N.B2_EINVAL and f"{fn}: sum_dy_xmu is not 4-byte aligned" in _err()


# ---- which inputs take the native path -----------------------------------------------------------------------------------
class _AnyDevice:
    """A CUDA device that compares equal to the CPU parameters' device, so a CPU layer can be routed without a GPU."""
    type, index = "cuda", 0

    def __eq__(self, other):
        return True

    def __ne__(self, other):
        return False


class _FakeCuda:
    """Just enough of a CUDA tensor for SyncBatchNorm.forward's checks and native_eligible."""

    def __init__(self, shape=(4, 16, 5, 5), dtype=torch.bfloat16, cl=True, ptr=P):
        self.shape, self.dtype, self._cl, self._ptr = shape, dtype, cl, ptr
        self.device, self.is_cuda, self.requires_grad = _AnyDevice(), True, True

    def dim(self):
        return len(self.shape)

    def size(self, i):
        return self.shape[i]

    def numel(self):
        n = 1
        for s in self.shape:
            n *= s
        return n

    def is_contiguous(self, memory_format=torch.contiguous_format):
        return self._cl if memory_format == torch.channels_last else not self._cl

    def data_ptr(self):
        return self._ptr


class _Comm:
    rank, device, ordered_stream = 0, 0, None

    def __init__(self, world):
        self.world = world


@pytest.fixture
def route(monkeypatch):
    """Runs a layer on a fake input with a stand-in communicator of `world` ranks; returns the path its forward took."""
    taken = []
    monkeypatch.setattr(B._SyncStats, "apply", lambda *a: taken.append("native") or (None, None, None))
    monkeypatch.setattr(B._SyncNormalise, "apply", lambda *a: "out")
    monkeypatch.setattr(B._FabricSyncBatchNorm, "apply", lambda *a: taken.append("aten") or "out")
    monkeypatch.setattr(B._NativeBatchNorm, "apply", lambda *a: taken.append("native_one_rank") or "out")
    monkeypatch.setattr(B.F, "batch_norm", lambda *a, **k: taken.append("F.batch_norm") or "out")

    def run(m, x, world=2):
        monkeypatch.setattr(D, "_COMM", _Comm(world))
        taken.clear()
        m(x)
        return taken[0]

    return run


def _layer(c=16, **kw):
    m = SyncBatchNorm(c, **kw)
    m.train()
    return m


def test_native_where_the_kernels_cover_the_input(route):
    assert route(_layer(), _FakeCuda()) == "native"
    assert route(_layer(momentum=None), _FakeCuda()) == "native"
    assert route(_layer(track_running_stats=False), _FakeCuda()) == "native"
    assert route(_layer(), _FakeCuda(shape=(2, 16, 1, 1))) == "native"  # two rows


def test_atens_compute_everywhere_else(route):
    for x in (_FakeCuda(dtype=torch.float16), _FakeCuda(dtype=torch.float32), _FakeCuda(cl=False), _FakeCuda(ptr=P + 2),
              _FakeCuda(shape=(1, 16, 1, 1)), _FakeCuda(shape=(0, 16, 5, 5)), _FakeCuda(shape=(4, 16, 25)),
              _FakeCuda(shape=(4, 16, 5, 5, 2)), _FakeCuda(shape=(8, 16))):
        assert route(_layer(), x) == "aten", (x.shape, x.dtype, x._cl, x._ptr)
    assert route(_layer(12), _FakeCuda(shape=(4, 12, 5, 5))) == "aten"  # C % 8 != 0
    assert route(_layer(affine=False), _FakeCuda()) == "aten"
    big = _FakeCuda(shape=(2**24, 128, 1, 1))  # 2^31 elements: ATen's reductions take another path
    assert route(_layer(128), big) == "aten"
    compiling = torch.compiler.is_compiling
    try:
        torch.compiler.is_compiling = lambda: True
        assert route(_layer(), _FakeCuda()) == "aten"
    finally:
        torch.compiler.is_compiling = compiling


def test_one_rank_takes_batchnorm2ds_native_path(route):
    assert route(_layer(), _FakeCuda(), world=1) == "native_one_rank"
    assert route(_layer(), _FakeCuda(cl=False), world=1) == "F.batch_norm"
    assert route(_layer(eps=0.0), _FakeCuda(), world=1) == "F.batch_norm"  # which refuses it, as before
    assert route(_layer(eps=0.0), _FakeCuda(), world=2) == "native"
    m = _layer()
    m.eval()
    assert route(m, _FakeCuda(), world=2) == "F.batch_norm"  # eval never synchronises


def test_hooks_do_not_change_the_layers_path(route):
    m = _layer()
    seen = []
    m.register_forward_pre_hook(lambda mod, inp: seen.append(1))
    assert route(m, _FakeCuda()) == "native" and seen == [1]


def test_under_a_process_group_it_is_torchs_module(monkeypatch):
    monkeypatch.setattr(D, "_COMM", _Comm(2))
    monkeypatch.setattr(D.dist, "is_initialized", lambda: True)
    assert not D._on_fabric()
    called = []
    monkeypatch.setattr(nn.SyncBatchNorm, "forward", lambda self, x: called.append(x) or "torch")
    assert _layer()(_FakeCuda()) == "torch" and len(called) == 1
    assert not _layer()._fusable()


def test_one_rank_on_cpu_tensors_is_f_batch_norm(monkeypatch):
    monkeypatch.setattr(D, "_COMM", None)
    torch.manual_seed(0)
    a, b = nn.BatchNorm2d(16), _layer()
    x = torch.randn(4, 16, 3, 3).to(memory_format=torch.channels_last)
    assert torch.equal(F.batch_norm(x, a.running_mean, a.running_var, a.weight, a.bias, True, 0.1, 1e-5), b(x))


# ---- fuse_resnet with SyncBatchNorm layers --------------------------------------------------------------------------------
torchvision = pytest.importorskip("torchvision")


def _block(bn_cls=None, **kw):
    from torchvision.models.resnet import BasicBlock

    blk = R.fuse_resnet(BasicBlock(16, 16))
    if bn_cls is not None:
        blk.bn1 = bn_cls(16, **kw)
        blk.bn2 = bn_cls(16, **kw)
    blk.train()
    return blk


def test_fusable_accepts_fabric_syncbatchnorm(monkeypatch):
    monkeypatch.setattr(D, "_COMM", _Comm(4))
    blk = SyncBatchNorm.convert_sync_batchnorm(_block())
    assert type(blk).__name__ == "FusedBasicBlock" and type(blk.bn1) is SyncBatchNorm
    assert R._fusable(blk, (blk.bn1, blk.bn2))
    assert R._two_phase(blk.bn1, _FakeCuda(dtype=torch.float32))  # over several ranks whatever the input
    monkeypatch.setattr(D, "_COMM", _Comm(1))
    assert R._fusable(blk, (blk.bn1, blk.bn2))
    assert not R._two_phase(blk.bn1, _FakeCuda(dtype=torch.float32)) and R._two_phase(blk.bn1, _FakeCuda())


def test_fusable_refuses_other_layers_and_states(monkeypatch):
    monkeypatch.setattr(D, "_COMM", _Comm(2))

    class MyBN(BatchNorm2d):
        pass

    class MySync(SyncBatchNorm):
        pass

    for cls in (MyBN, MySync, nn.SyncBatchNorm, nn.BatchNorm2d):
        blk = _block(cls)
        assert not R._fusable(blk, (blk.bn1, blk.bn2)), cls
    blk = _block(SyncBatchNorm)
    assert R._fusable(blk, (blk.bn1, blk.bn2))
    blk.bn1.eval()
    assert not R._fusable(blk, (blk.bn1, blk.bn2))
    blk = _block(SyncBatchNorm, eps=0.0)
    assert not R._fusable(blk, (blk.bn1, blk.bn2))
    assert not R._fusable(_block(SyncBatchNorm, affine=False), (_block(SyncBatchNorm, affine=False).bn1,))
    half = _block(SyncBatchNorm)
    half.bn2.running_var = half.bn2.running_var.half()
    assert not R._fusable(half, (half.bn1, half.bn2))
    grouped = _block(SyncBatchNorm, process_group=object())  # not a B200Group: refused in forward, never fused
    assert not R._fusable(grouped, (grouped.bn1, grouped.bn2))
    hooked = _block(SyncBatchNorm)
    hooked.bn2.register_forward_hook(lambda *a: None)
    assert not R._fusable(hooked, (hooked.bn1, hooked.bn2))
    monkeypatch.setattr(D, "_COMM", None)  # off the fabric: torch's module
    blk = _block(SyncBatchNorm)
    assert not R._fusable(blk, (blk.bn1, blk.bn2))
