"""The native BatchNorm2d reductions, the parts that need no GPU: the host restates ATen's launch geometry for its
channels-last reductions (flexible_launch_configs with coop = true), which fixes the reduction order per channel; every
argument check of b2_bn_stats / b2_bn_backward_reduce; and which inputs take the native reductions."""
import ctypes
import os
import re

import pytest
import torch

from torchx_b200.ddp import _native as N
from torchx_b200.nn import bn2d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# [M, C] of ResNet-50's BatchNorm layers at B = 256, the odd shapes of the bit-equality tests, and shapes at the edges of
# flexible_launch_configs' branches (block_y < 16, grid_y raised to 1 below 8, grid_y 8..15, the 128 cap, C not a power of 2)
RESNET50 = [(256 * h * w, c) for (_, c, h, w) in [(256, 64, 112, 112), (256, 256, 56, 56), (256, 512, 28, 28), (256, 128, 56, 56),
                                                   (256, 1024, 14, 14), (256, 256, 28, 28), (256, 64, 56, 56), (256, 2048, 7, 7),
                                                   (256, 128, 28, 28), (256, 512, 14, 14), (256, 256, 14, 14), (256, 512, 7, 7)]]
ODD = [(2, 8), (3, 24), (7, 72), (12545, 8), (12545, 24), (12545, 72)]
BOUNDARY = [(2, 64), (3, 64), (7, 64), (16, 64), (17, 64), (255, 64), (256, 64), (257, 64), (1024, 64), (1792, 64), (1793, 64),
            (2560, 64), (4096, 64), (4097, 64), (32768, 64), (32769, 64), (12544, 2048), (12545, 1000), (5000, 24), (5000, 72),
            (100000, 8), (100000, 16), (268435455, 8), (33554431, 64)]
SHAPES = RESNET50 + ODD + BOUNDARY


def _last_pow2(n):
    """ATen's lastPow2 (LaunchUtils.h)."""
    for s in (1, 2, 4, 8, 16):
        n |= n >> s
    return max(1, n - (n >> 1))


def _flexible_launch_configs(reduction, stride):
    """ATen's flexible_launch_configs(reduction, stride, block, grid, coop_flag=true) (Normalization.cuh)."""
    block_x = min(_last_pow2(stride), 32)
    block_y = min(_last_pow2(-(-reduction // 16)), 512 // block_x)
    if block_x * block_y != 512:
        block_x = min(_last_pow2(stride), 512 // block_y)
    grid_x = -(-stride // block_x)
    grid_y = min(-(-reduction // (block_y * 16)), 128)
    grid_y = 1 if grid_y < 8 else grid_y
    return block_x, block_y, grid_x, grid_y


def _plan(rows, channels):
    geom, nbytes = (ctypes.c_int * 4)(), ctypes.c_size_t()
    rc = N.lib().b2_bn_reduce_plan(rows, channels, geom, ctypes.byref(nbytes))
    return rc, tuple(geom), nbytes.value


@pytest.mark.parametrize("M,C", SHAPES, ids=[f"M{m}xC{c}" for m, c in SHAPES])
def test_host_geometry_is_atens(M, C):
    rc, geom, nbytes = _plan(M, C)
    assert rc == N.B2_OK
    assert geom == _flexible_launch_configs(M, C)
    _, block_y, _, grid_y = geom
    # ATen's backward reduce returns early from threads with m_offset >= M; there are none, so no valid channel misses a chain
    assert block_y * grid_y <= M
    assert nbytes == (grid_y * (2 * C + C // 8) * 4 if grid_y > 1 else 0)


def test_the_branches_are_covered():
    geoms = {s: _flexible_launch_configs(*s) for s in SHAPES}
    assert any(g[3] == 1 and g[1] < 16 for g in geoms.values())  # grid_y == 1, block_y < 16
    assert _flexible_launch_configs(1024, 64)[3] == 1 and -(-1024 // (16 * 16)) in range(2, 8)  # grid_y raised to 1
    assert 8 <= _flexible_launch_configs(2560, 64)[3] <= 15 and _flexible_launch_configs(2560, 64)[1] == 16  # grid_y < block_y
    assert _flexible_launch_configs(12544, 2048)[3] == 49
    assert _flexible_launch_configs(802816, 64)[3] == 128  # the cap
    assert any(M % (g[1] * g[3] * 4) for (M, _), g in geoms.items())  # ragged rows per sequence


# ---- C ABI -------------------------------------------------------------------------------------------------------------
def test_header_declares_the_entry_points_and_the_binding_resolves_them():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    assert re.search(r"int b2_bn_reduce_plan\(size_t rows, size_t channels, int\* geometry, size_t\* workspace_bytes\);", src)
    assert re.search(r"int b2_bn_stats\(const void\* x, size_t rows, size_t channels, int dtype, float\* mean, float\* var,", src)
    assert re.search(r"int b2_bn_backward_reduce\(const void\* dy, const void\* x, size_t rows, size_t channels, int dtype,", src)
    L = N.lib()
    for name, nargs in (("b2_bn_reduce_plan", 4), ("b2_bn_stats", 13), ("b2_bn_backward_reduce", 15)):
        assert name in N.SYMBOLS
        assert getattr(L, name).restype is ctypes.c_int and len(getattr(L, name).argtypes) == nargs


def _err():
    return N.lib().b2_last_error().decode()


P = 1 << 20  # an aligned fake device address: every call below fails validation before anything touches it


def _stats(x=P, rows=64, channels=16, dtype=N.B2_DT_BFLOAT16, mean=P, var=P, rm=P, rv=P, ws=None, ws_bytes=0):
    return N.lib().b2_bn_stats(x, rows, channels, dtype, mean, var, rm, rv, 0.1, ws, ws_bytes, 0, None)


def _reduce(dy=P, x=P, rows=64, channels=16, dtype=N.B2_DT_BFLOAT16, mean=P, invstd=P, sum_dy=P, sum_dy_xmu=P, gw=P, gb=P, ws=None,
            ws_bytes=0):
    return N.lib().b2_bn_backward_reduce(dy, x, rows, channels, dtype, mean, invstd, sum_dy, sum_dy_xmu, gw, gb, ws, ws_bytes, 0, None)


@pytest.mark.parametrize("call,fn", [(_stats, "b2_bn_stats"), (_reduce, "b2_bn_backward_reduce")])
def test_validation_messages(call, fn):
    for dtype in (N.B2_DT_FLOAT16, N.B2_DT_FLOAT32, 7):
        assert call(dtype=dtype) == N.B2_EINVAL
        assert f"{fn}: dtype {dtype} is not B2_DT_BFLOAT16" in _err()
    for c in (0, 12):
        assert call(channels=c) == N.B2_EINVAL
        assert f"{fn}: channels={c} must be a positive multiple of 8" in _err()
    for rows in (0, 1):
        assert call(rows=rows) == N.B2_EINVAL
        assert f"{fn}: rows={rows}, batch statistics need at least 2" in _err()
    for rows, c in ((268435456, 8), (33554432, 64), (1 << 40, 8)):
        assert call(rows=rows, channels=c) == N.B2_EINVAL
        assert f"{fn}: rows*channels={rows} x {c} must be below 2^31 - 1 elements" in _err()
    assert call(x=None) == N.B2_EINVAL and f"{fn}: null x" in _err()
    assert call(x=P + 8) == N.B2_EINVAL and f"{fn}: x is not 16-byte aligned" in _err()
    assert call(mean=None) == N.B2_EINVAL and f"{fn}: null mean" in _err()
    assert call(mean=P + 2) == N.B2_EINVAL and f"{fn}: mean is not 4-byte aligned" in _err()
    # a layer whose tree has several CTA rows needs the workspace b2_bn_reduce_plan reports
    rows, c = 2560, 64
    _, (_, _, _, grid_y), need = _plan(rows, c)
    assert grid_y == 10 and need == 10 * (2 * 64 + 8) * 4
    assert call(rows=rows, channels=c) == N.B2_EINVAL and f"{fn}: null workspace ({need} bytes needed)" in _err()
    assert call(rows=rows, channels=c, ws=P + 2, ws_bytes=need) == N.B2_EINVAL and f"{fn}: workspace is not 4-byte aligned" in _err()
    assert call(rows=rows, channels=c, ws=P, ws_bytes=need - 4) == N.B2_EINVAL
    assert f"{fn}: workspace of {need - 4} bytes, {need} needed" in _err()


def test_validation_of_the_pass_specific_pointers():
    assert _stats(var=None) == N.B2_EINVAL and "b2_bn_stats: null var" in _err()
    for rm, rv in ((P, None), (None, P)):
        assert _stats(rm=rm, rv=rv) == N.B2_EINVAL
        assert "b2_bn_stats: running_mean and running_var must both be given or both be null" in _err()
    assert _stats(rm=P + 1) == N.B2_EINVAL and "b2_bn_stats: running_mean is not 4-byte aligned" in _err()
    assert _stats(rv=P + 2) == N.B2_EINVAL and "b2_bn_stats: running_var is not 4-byte aligned" in _err()
    assert _reduce(dy=None) == N.B2_EINVAL and "b2_bn_backward_reduce: null dy" in _err()
    assert _reduce(dy=P + 8) == N.B2_EINVAL and "b2_bn_backward_reduce: dy is not 16-byte aligned" in _err()
    assert _reduce(invstd=None) == N.B2_EINVAL and "b2_bn_backward_reduce: null invstd" in _err()
    assert _reduce(sum_dy=P + 2) == N.B2_EINVAL and "b2_bn_backward_reduce: sum_dy is not 4-byte aligned" in _err()
    assert _reduce(sum_dy_xmu=None) == N.B2_EINVAL and "b2_bn_backward_reduce: null sum_dy_xmu" in _err()
    assert _reduce(gw=None) == N.B2_EINVAL and "b2_bn_backward_reduce: null grad_weight" in _err()
    assert _reduce(gb=P + 1) == N.B2_EINVAL and "b2_bn_backward_reduce: grad_bias is not 4-byte aligned" in _err()


def test_plan_validation():
    geom, nbytes = (ctypes.c_int * 4)(), ctypes.c_size_t()
    assert N.lib().b2_bn_reduce_plan(64, 12, geom, ctypes.byref(nbytes)) == N.B2_EINVAL
    assert "b2_bn_reduce_plan: channels=12 must be a positive multiple of 8" in _err()
    assert N.lib().b2_bn_reduce_plan(1, 8, geom, ctypes.byref(nbytes)) == N.B2_EINVAL
    assert N.lib().b2_bn_reduce_plan(268435456, 8, geom, ctypes.byref(nbytes)) == N.B2_EINVAL
    assert N.lib().b2_bn_reduce_plan(64, 8, None, ctypes.byref(nbytes)) == N.B2_EINVAL
    assert "b2_bn_reduce_plan: null geometry or workspace_bytes" in _err()


# ---- which inputs take the native reductions ----------------------------------------------------------------------------
class _Numel:
    def __init__(self, n):
        self.n = n

    def numel(self):
        return self.n


def test_native_reductions_follow_atens_32_bit_index_check():
    assert bn2d.native_reductions(_Numel(2**31 - 2))
    assert not bn2d.native_reductions(_Numel(2**31 - 1))
    assert not bn2d.native_reductions(_Numel(2**31))
    assert bn2d.native_reductions(torch.empty(2, 8, 1, 1))
