"""SyncBatchNorm on the native communicator, the parts that need no GPU: the C ABI entry and its argument checks, the numpy
restatement of ATen's statistics merge (tests/_bn_oracle.py) against a float64 Welford, convert_sync_batchnorm, the
module off the fabric, and what it refuses on the fabric."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
from torch import nn

import torchx_b200.distributed as D
from tests import _bn_oracle as O
from torchx_b200.ddp import _native as N
from torchx_b200.nn import SyncBatchNorm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- C ABI -------------------------------------------------------------------------------------------------------------
def test_header_declares_the_entry_point_and_the_binding_resolves_it():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    assert re.search(r"int b2_batchnorm_stats\(b2_comm_t\* comm, float\* mean, float\* invstd, float count, size_t channels,\s*"
                     r"float\* running_mean, float\* running_var, double momentum, double eps,\s*float\* counts_out, void\* stream\);",
                     src)
    assert int(re.search(r"#define\s+B2_ABI_VERSION\s+(\d+)", src).group(1)) == N.B2_ABI_VERSION == 3
    assert "b2_batchnorm_stats" in N.SYMBOLS
    L = N.lib()
    assert hasattr(L, "b2_batchnorm_stats") and L.b2_batchnorm_stats.restype is ctypes.c_int
    assert len(L.b2_batchnorm_stats.argtypes) == 11


def test_argument_validation_without_a_gpu():
    L = N.lib()
    p = ctypes.c_void_p(4096)
    call = lambda mean, invstd, count, channels, comm=None: L.b2_batchnorm_stats(  # noqa: E731
        comm, mean, invstd, count, channels, None, None, 0.1, 1e-5, None, None)
    assert call(None, None, float("nan"), 0) == N.B2_OK  # channels == 0: a no-op, nothing is read
    for mean, invstd in ((None, p), (p, None)):
        assert call(mean, invstd, 4.0, 3) == N.B2_EINVAL
        assert b"b2_batchnorm_stats: null mean or invstd" in L.b2_last_error()
    for bad in (-1.0, float("nan"), -float("inf")):
        assert call(p, p, bad, 3) == N.B2_EINVAL, bad
        assert b"b2_batchnorm_stats: count must be >= 0" in L.b2_last_error(), bad
    assert call(p, p, 4.0, 3) == N.B2_EINVAL  # no communicator
    assert b"null communicator" in L.b2_last_error()


# ---- the merge -------------------------------------------------------------------------------------------------------
def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a, b, c = (rng.standard_normal(2000).astype(np.float32) for _ in range(3))
    c[:500] = -(a[:500].astype(np.float64) * b[:500]).astype(np.float32)  # cancellation: the error term decides
    from fractions import Fraction

    got = O.fma32(a, b, c)
    for i in range(0, 2000, 7):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        # the correctly rounded fp32 of `exact`: the nearer of the two fp32 neighbours of float(exact), ties to even
        x = np.float32(float(exact))
        lo, hi = sorted({x, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(-np.inf))},
                        key=lambda y: abs(Fraction(float(y)) - exact))[:2]
        da, db = abs(Fraction(float(lo)) - exact), abs(Fraction(float(hi)) - exact)
        want = lo if da < db else (hi if db < da else (lo if (lo.view(np.uint32) & 1) == 0 else hi))
        assert got[i] == want, (i, a[i], b[i], c[i], got[i], want)


@pytest.mark.parametrize("sizes", [[64, 64], [17, 200, 3], [1, 1, 1, 1], [5, 0, 30, 0, 9, 120, 2, 41]])
def test_merge_matches_a_float64_welford(sizes):
    """The merged mean and invstd are within 4e-6 relative (a few fp32 ulps of the result's scale) of the fp64 statistics
    of the concatenated batch; the running variance uses the unbiased estimate."""
    rng = np.random.default_rng(len(sizes))
    C, eps, mom = 37, 1e-5, 0.1
    xs = [(rng.standard_normal((n, C)) * rng.uniform(0.5, 3, C) + rng.uniform(-2, 2, C)).astype(np.float32) for n in sizes]
    rows = [O.local_stats(x, eps) if x.shape[0] else (np.zeros(C, np.float32), np.zeros(C, np.float32), np.float32(0))
            for x in xs]
    rm0, rv0 = rng.standard_normal(C).astype(np.float32), rng.uniform(0.5, 2, C).astype(np.float32)
    mean, invstd, rm, rv = O.gather_stats([r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], rm0, rv0, mom, eps)
    allx = np.concatenate(xs).astype(np.float64)
    m64, v64 = allx.mean(0), allx.var(0)
    scale = np.sqrt(v64) + np.abs(m64)
    assert np.all(np.abs(mean - m64) <= 4e-6 * scale)
    assert np.allclose(invstd, 1 / np.sqrt(v64 + eps), rtol=4e-5, atol=0)
    assert np.allclose(rm, (1 - mom) * rm0 + mom * m64, rtol=1e-5, atol=1e-6)
    n = allx.shape[0]
    unbiased = v64 * n / (n - 1) if n > 1 else np.full(C, np.inf)
    assert np.allclose(rv, (1 - mom) * rv0 + mom * unbiased, rtol=1e-4, atol=1e-6)


def test_one_rank_alone_gives_back_its_own_statistics():
    """With a power-of-two count the mean comes back bit for bit; invstd goes through 1/invstd, ^2, - eps, + eps, sqrt
    and a reciprocal, so it comes back within a few ulps."""
    rng = np.random.default_rng(3)
    m = rng.standard_normal(100).astype(np.float32)
    s = rng.uniform(0.1, 10, 100).astype(np.float32)
    for cnt in (1, 2, 64, 1 << 20):
        mean, invstd, _, _ = O.gather_stats([m], [s], [cnt])
        assert mean.view(np.uint32).tolist() == m.view(np.uint32).tolist(), cnt
        assert np.max(np.abs(invstd.view(np.int32) - s.view(np.int32))) <= 4, cnt
    mean, invstd, _, _ = O.gather_stats([m], [s], [37])  # 37 * fl(1/37) rounds: within an ulp
    assert np.max(np.abs(mean.view(np.int32) - m.view(np.int32))) <= 1


def test_zero_count_ranks_are_left_out():
    rng = np.random.default_rng(5)
    C = 50
    means = rng.standard_normal((3, C)).astype(np.float32)
    invs = rng.uniform(0.5, 2, (3, C)).astype(np.float32)
    counts = np.array([12, 7, 300], np.float32)
    rm, rv = rng.standard_normal(C).astype(np.float32), rng.uniform(0.5, 2, C).astype(np.float32)
    want = O.gather_stats(means, invs, counts, rm, rv, 0.3, 1e-3)
    junk = rng.standard_normal((2, C)).astype(np.float32) * 1e6  # what an empty rank's row holds does not matter
    for at in ([0, 0], [1, 3], [3, 3]):  # positions in the original 3 rows
        m2 = np.insert(means, at, junk, axis=0)
        i2 = np.insert(invs, at, junk, axis=0)
        c2 = np.insert(counts, at, [0, 0.5])  # below one sample: torch's mask drops it
        got = O.gather_stats(m2, i2, c2, rm, rv, 0.3, 1e-3)
        for g, w in zip(got, want):
            assert g.view(np.uint32).tolist() == w.view(np.uint32).tolist(), at


def test_an_all_empty_world_gives_torchs_masked_result():
    """torch's mask leaves no row: ATen's loop runs zero times, so mean = 0, invstd = 1 / sqrt(0 / 0 + eps) = NaN, and the
    running statistics decay towards 0 (running_var by momentum * (0 / -1) = -0)."""
    C = 8
    rm = np.linspace(-1, 1, C).astype(np.float32)
    rv = np.linspace(0.5, 2, C).astype(np.float32)
    mean, invstd, grm, grv = O.gather_stats(np.ones((2, C), np.float32), np.ones((2, C), np.float32), [0, 0], rm, rv, 0.1, 1e-5)
    assert (mean == 0).all() and not np.signbit(mean).any()
    assert np.isnan(invstd).all()
    om = np.float32(1) - np.float32(0.1)
    assert grm.tolist() == (om * rm).tolist() and grv.tolist() == (om * rv).tolist()


# ---- convert_sync_batchnorm --------------------------------------------------------------------------------------------
def _net(**bn):
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8, **bn), nn.ReLU(),
                         nn.Sequential(nn.Linear(4, 4), nn.BatchNorm1d(6, **bn), nn.Sequential(nn.BatchNorm3d(5, **bn))))


@pytest.mark.parametrize("bn", [{}, {"affine": False}, {"track_running_stats": False}, {"momentum": None}, {"eps": 1e-3}])
def test_convert_matches_torchs_conversion(bn):
    ours = SyncBatchNorm.convert_sync_batchnorm(_net(**bn))
    theirs = nn.SyncBatchNorm.convert_sync_batchnorm(_net(**bn))
    converted = [m for m in ours.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)]
    assert len(converted) == 3 and all(type(m) is SyncBatchNorm for m in converted)
    assert all(isinstance(m, nn.SyncBatchNorm) for m in converted)
    for a, b in zip(converted, (m for m in theirs.modules() if isinstance(m, nn.SyncBatchNorm))):
        assert (a.num_features, a.eps, a.momentum, a.affine, a.track_running_stats) == \
               (b.num_features, b.eps, b.momentum, b.affine, b.track_running_stats)
    so, st = ours.state_dict(), theirs.state_dict()
    assert list(so) == list(st)
    for k in so:
        assert so[k].dtype == st[k].dtype and torch.equal(so[k], st[k]), k
    theirs.load_state_dict(so)
    ours.load_state_dict(st)


def test_convert_shares_parameters_and_buffers_and_copies_flags():
    bn = nn.BatchNorm2d(4)
    bn.weight.requires_grad_(False)
    bn.num_batches_tracked.fill_(7)
    bn.eval()
    bn.qconfig = "marker"
    out = SyncBatchNorm.convert_sync_batchnorm(bn, process_group=None)
    assert type(out) is SyncBatchNorm
    assert out.weight is bn.weight and out.bias is bn.bias
    assert out.running_mean is bn.running_mean and out.running_var is bn.running_var
    assert out.num_batches_tracked is bn.num_batches_tracked and int(out.num_batches_tracked) == 7
    assert out.weight.requires_grad is False and out.bias.requires_grad is True
    assert out.training is False and out.qconfig == "marker"


def test_convert_takes_torch_syncbatchnorm_layers_too():
    torch_sbn = nn.SyncBatchNorm.convert_sync_batchnorm(_net())
    ours = SyncBatchNorm.convert_sync_batchnorm(torch_sbn)
    assert [type(m) for m in ours.modules() if isinstance(m, nn.SyncBatchNorm)] == [SyncBatchNorm] * 3
    again = SyncBatchNorm.convert_sync_batchnorm(ours)  # already converted: left as it is
    assert [m for m in again.modules()] == [m for m in ours.modules()]


# ---- the module off the fabric -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(6, 4), (5, 4, 3, 3)])
@pytest.mark.parametrize("bn", [{}, {"momentum": None}, {"track_running_stats": False}])
def test_off_the_fabric_it_is_torchs_fallback(shape, bn):
    """No process group and no communicator: torch's SyncBatchNorm runs F.batch_norm, and so does ours, bit for bit, in
    training and in eval mode."""
    assert not D._on_fabric()
    torch.manual_seed(1)
    a, b = nn.SyncBatchNorm(4, **bn), SyncBatchNorm(4, **bn)
    b.load_state_dict(a.state_dict())
    for train in (True, True, False):
        a.train(train)
        b.train(train)
        x = torch.randn(*shape)
        assert torch.equal(a(x), b(x))
        for k, v in a.state_dict().items():
            assert torch.equal(v, b.state_dict()[k]), k


# ---- refusals on the fabric --------------------------------------------------------------------------------------------
class _FakeComm:
    rank, world, device, ordered_stream = 0, 2, 0, None


@pytest.fixture
def on_fabric(monkeypatch):
    monkeypatch.setattr(D, "_COMM", _FakeComm())
    assert D._on_fabric()


def test_refusals_on_the_fabric(on_fabric):
    x = torch.randn(4, 3, 2, 2)
    with pytest.raises(ValueError, match="expected input tensor to be on GPU"):
        SyncBatchNorm(3)(x)
    with pytest.raises(NotImplementedError, match="no subgroups"):
        SyncBatchNorm(3, process_group=object())(x)
    with pytest.raises(TypeError, match="float32 running statistics"):
        SyncBatchNorm(3).double()(x.double())
    with pytest.raises(TypeError, match="float32 running statistics"):
        SyncBatchNorm(3).half()(x.half())


def test_eval_mode_on_the_fabric_is_torchs_fallback(on_fabric):
    """eval mode never synchronises: it normalises with the running statistics, whatever device the input is on."""
    torch.manual_seed(2)
    a, b = nn.SyncBatchNorm(3), SyncBatchNorm(3)
    a.running_mean.uniform_(-1, 1)
    a.running_var.uniform_(0.5, 2)
    b.load_state_dict(a.state_dict())
    a.eval()
    b.eval()
    x = torch.randn(4, 3, 5)
    assert torch.equal(a(x), b(x))


def test_binding_rejects_non_float32_tensors_before_the_library():
    from torchx_b200.ddp import Communicator

    c = Communicator.__new__(Communicator)  # no handle: the dtype check comes before anything reaches the library
    c.world, c.device = 2, 0
    t32, t16 = torch.zeros(4), torch.zeros(4, dtype=torch.float16)
    for kw in ({"mean": t16, "invstd": t32}, {"mean": t32, "invstd": t16}, {"mean": t32, "invstd": t32, "running_mean": t16},
               {"mean": t32, "invstd": t32, "running_var": t16}):
        mean, invstd = kw.pop("mean"), kw.pop("invstd")
        with pytest.raises(TypeError, match="must be float32"):
            c.batchnorm_stats_(mean, invstd, 3.0, momentum=0.1, eps=1e-5, **kw)
    with pytest.raises(TypeError, match="counts_out must be float32"):
        c.batchnorm_stats_(t32, t32, 3.0, momentum=0.1, eps=1e-5, counts_out=torch.zeros(2, dtype=torch.int32))
