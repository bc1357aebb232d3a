"""The native BatchNorm2d reductions on the GPU: an eligible layer runs k_bn2d_stats / k_bn2d_bwd_reduce instead of ATen's
channels-last reductions, and the converted layer stays bit-equal to nn.BatchNorm2d at shapes that reach every branch of
ATen's reduction tree, with constant channels, and where a padding slot follows an inf (the slot's update turns an infinite
mean or sum into NaN, as ATen's does); an input of 2^31 elements or more keeps ATen's reductions; reruns are bit-identical."""
import copy

import pytest
import torch

from tests.test_native_bn_gpu import _assert_same_bits, _inputs, _run, _step
from tests.test_native_bn_reduce import _flexible_launch_configs
from torchx_b200.ddp import _native as N
from torchx_b200.nn import BatchNorm2d, bn2d, convert_batchnorm

pytestmark = pytest.mark.gpu

ATEN_REDUCTIONS = ("batch_norm_collect_statistics", "batch_norm_backward_reduce")


def _kernel_names(bn, x, dy):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _step(bn, x, dy)
        torch.cuda.synchronize()
    return " ".join(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


@pytest.mark.parametrize("shape", [(4, 64, 16, 16), (10, 64, 16, 16)], ids=["grid_y1", "grid_y10"])
def test_eligible_layers_launch_no_aten_reduction(shape):
    x, dy, ref = _inputs(shape, torch.bfloat16, 29)
    names = _kernel_names(convert_batchnorm(ref), x, dy)
    assert "k_bn2d_stats" in names and "k_bn2d_bwd_reduce" in names
    assert ("k_bn2d_stats_merge" in names) == (shape[0] == 10) and ("k_bn2d_bwd_reduce_merge" in names) == (shape[0] == 10)
    for aten in ATEN_REDUCTIONS:
        assert aten not in names


def test_ineligible_layers_keep_atens_reductions():
    # bf16 channels-last with C % 8 != 0: ATen's own channels-last kernels (an fp32 input would run cuDNN's BatchNorm)
    x, dy, ref = _inputs((8, 12, 16, 16), torch.bfloat16, 31)
    bn = convert_batchnorm(ref)
    assert not bn2d.native_eligible(bn, x)
    names = _kernel_names(bn, x, dy)
    assert "k_bn2d_" not in names
    for aten in ATEN_REDUCTIONS:
        assert aten in names


# (N, C, H, W), each reaching one branch of flexible_launch_configs / the merge tree
BRANCHES = {
    "M2_block_y1": (2, 64, 1, 1),
    "M3_block_y1": (3, 64, 1, 1),
    "M7_block_y1": (7, 64, 1, 1),
    "M1024_grid_y4_raised_to_1": (4, 64, 16, 16),
    "M2560_grid_y10_below_block_y": (10, 64, 16, 16),
    "M4551_ragged": (3, 64, 37, 41),
    "M12544xC2048_grid_y49": (256, 2048, 7, 7),
    "C24": (4, 24, 33, 35),
    "C72": (4, 72, 33, 35),
    "C1000": (2, 1000, 50, 63),
    "M802816xC64_grid_y128": (256, 64, 56, 56),
}


@pytest.mark.parametrize("shape", list(BRANCHES.values()), ids=list(BRANCHES))
def test_branches_are_bit_equal(shape):
    _run(shape, torch.bfloat16, seed=37)


def test_constant_channel_is_bit_equal():
    shape = (3, 64, 37, 41)
    x, dy, ref = _inputs(shape, torch.bfloat16, 41)
    x[:, 5] = 3.0
    x[:, 6] = 0.0
    dy[:, 7] = -0.0
    mine = convert_batchnorm(copy.deepcopy(ref))
    _assert_same_bits(_step(ref, x, dy), _step(mine, x, dy))


def _rows_before_padding(M, C):
    """Rows r whose chain's next row, r + 4*S, is past M while the chain still has an iteration left: in ATen (and here)
    the update after r is a padding slot with x = 0, 1/count = 0, is_valid = 0."""
    _, block_y, _, grid_y = _flexible_launch_configs(M, C)
    S = block_y * grid_y
    loops = 1 + (M - 1) // (4 * S)
    return [r for r in range(M) if (r // S) // 4 == loops - 2 and r + 4 * S >= M]


def _nhw(shape, row):
    _, _, h, w = shape
    n, r = divmod(row, h * w)
    return n, r // w, r % w


PADDED = {"M4551_grid_y18": (3, 64, 37, 41), "M1000_grid_y1": (1, 64, 25, 40)}


@pytest.mark.parametrize("shape", list(PADDED.values()), ids=list(PADDED))
def test_padding_slot_after_an_inf_turns_the_mean_into_nan(shape):
    # An inf makes the chain's mean inf; the padding slot after it computes mean = FFMA(0 - inf, 0, inf) = NaN.  A kernel
    # that skipped padding slots would leave the channel's mean inf.
    n, c, h, w = shape
    rows = _rows_before_padding(n * h * w, c)
    assert len(rows) >= 2
    x, dy, ref = _inputs(shape, torch.bfloat16, 43)
    x[(_nhw(shape, rows[0])[0], 3) + _nhw(shape, rows[0])[1:]] = float("inf")
    x[(_nhw(shape, rows[-1])[0], 9) + _nhw(shape, rows[-1])[1:]] = -float("inf")
    dy[(_nhw(shape, rows[1])[0], 10) + _nhw(shape, rows[1])[1:]] = float("inf")
    mine = convert_batchnorm(copy.deepcopy(ref))
    a, b = _step(ref, x, dy), _step(mine, x, dy)
    _assert_same_bits(a, b)
    assert torch.isnan(b["mean"][3]) and torch.isnan(b["mean"][9])
    assert torch.isfinite(b["mean"][0]) and not torch.isfinite(b["gb"][10])


@pytest.mark.parametrize("shape", list(PADDED.values()), ids=list(PADDED))
def test_backward_padding_slot_with_an_infinite_mean_gives_nan(shape):
    # With mean = +inf and dy > 0 every valid term of sum_dy_xmu is -inf; the padding slots add FFMA(0 - inf, 0, s) = NaN,
    # so ATen's sum is NaN where a kernel that skipped them would give -inf.  Called directly: the layer's own mean is NaN.
    n, c, h, w = shape
    M = n * h * w
    x, dy, _ = _inputs(shape, torch.bfloat16, 59)
    dy = dy.abs() + 0.5
    mean = torch.zeros(c, device="cuda")
    mean[5] = float("inf")
    invstd = torch.ones(c, device="cuda")
    weight = torch.ones(c, device="cuda")
    want = torch.batch_norm_backward_reduce(dy, x, mean, invstd, weight, True, True, True)
    got = [torch.empty(c, device="cuda") for _ in range(4)]
    ws, ws_bytes = bn2d._workspace(M, c, x.device)
    N.check(N.lib().b2_bn_backward_reduce(dy.data_ptr(), x.data_ptr(), M, c, N.B2_DT_BFLOAT16, mean.data_ptr(), invstd.data_ptr(),
                                          *(t.data_ptr() for t in got), bn2d._ptr(ws), ws_bytes, x.device.index,
                                          torch.cuda.current_stream().cuda_stream))
    _assert_same_bits(dict(zip("abcd", want)), dict(zip("abcd", got)))
    assert torch.isnan(got[1][5]) and torch.isfinite(got[1][4])


def test_two_runs_are_bit_identical():
    shape = (256, 64, 56, 56)
    outs = []
    for _ in range(2):
        x, dy, ref = _inputs(shape, torch.bfloat16, 47)
        outs.append(_step(convert_batchnorm(ref), x, dy))
    _assert_same_bits(outs[0], outs[1])


def test_input_of_2_31_elements_stays_on_atens_reductions():
    n, c, h, w = 128, 64, 512, 512  # 2^31 elements: beyond ATen's 32-bit index check
    # x and dy stay, the step adds an input clone, y and dx (4 GiB each in bf16) and ATen's temporaries; each step's y and
    # dx go to host memory before the next one, so at most about 24 GiB of device memory are in use at once
    if torch.cuda.mem_get_info()[0] < 32 * 2**30:
        pytest.skip("needs 32 GiB of free device memory")
    g = torch.Generator(device="cuda").manual_seed(53)
    x = torch.randn(n, h, w, c, device="cuda", dtype=torch.bfloat16, generator=g).permute(0, 3, 1, 2)
    dy = torch.randn(n, h, w, c, device="cuda", dtype=torch.bfloat16, generator=g).permute(0, 3, 1, 2)
    assert x.is_contiguous(memory_format=torch.channels_last) and not bn2d.native_reductions(x)
    ref = torch.nn.BatchNorm2d(c).cuda()
    mine = convert_batchnorm(copy.deepcopy(ref))
    assert type(mine) is BatchNorm2d and bn2d.native_eligible(mine, x)
    outs = []
    for bn in (ref, mine):
        out = _step(bn, x, dy)
        outs.append({k: v.cpu() for k, v in out.items()})
        del out
        torch.cuda.empty_cache()
    _assert_same_bits(*outs)
