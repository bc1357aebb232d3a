"""Native BatchNorm2d on the GPU: on bf16 the converted layer computes the bits nn.BatchNorm2d computes (DESIGN.md 2.4) - outputs,
input / weight / bias gradients, saved mean / invstd and running statistics - at ResNet-50's shapes, odd shapes, large
offsets and non-finite inputs; reruns are bit-identical; and the mini-DDP's converted layers run in a training step."""
import copy

import pytest
import torch
from torch import nn

from torchx_b200.nn import BatchNorm2d, convert_batchnorm

pytestmark = pytest.mark.gpu

# [M = N*H*W, C] of ResNet-50's 53 BatchNorm layers at B = 256, as (N, C, H, W)
RESNET50 = [(256, 64, 112, 112), (256, 256, 56, 56), (256, 512, 28, 28), (256, 128, 56, 56), (256, 1024, 14, 14), (256, 256, 28, 28),
            (256, 64, 56, 56), (256, 2048, 7, 7), (256, 128, 28, 28), (256, 512, 14, 14), (256, 256, 14, 14), (256, 512, 7, 7)]
ODD = [(2, 8, 1, 1), (3, 24, 1, 1), (7, 72, 1, 1), (5, 8, 13, 193), (5, 24, 13, 193), (5, 72, 13, 193)]
KEYS = ("y", "dx", "gw", "gb", "mean", "invstd", "rm", "rv")


def _inputs(shape, dtype, seed, offset=0.0, scale=1.0, **bn_kw):
    g = torch.Generator(device="cuda").manual_seed(seed)
    n, c, h, w = shape
    x = (torch.randn(shape, device="cuda", generator=g) * scale + offset).to(dtype).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(shape, device="cuda", generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
    ref = nn.BatchNorm2d(c, **bn_kw).cuda()
    with torch.no_grad():
        ref.weight.uniform_(0.5, 1.5, generator=g)
        ref.bias.uniform_(-0.5, 0.5, generator=g)
        if ref.track_running_stats:
            ref.running_mean.uniform_(-1.0, 1.0, generator=g)
            ref.running_var.uniform_(0.5, 2.0, generator=g)
    return x, dy, ref


def _step(bn, x, dy):
    xi = x.detach().clone().requires_grad_()
    y = bn(xi)
    mean, invstd = _saved_stats(y)
    y.backward(dy)
    out = {"y": y.detach(), "dx": xi.grad, "gw": bn.weight.grad.clone(), "gb": bn.bias.grad.clone(), "mean": mean, "invstd": invstd}
    if bn.track_running_stats:
        out.update(rm=bn.running_mean.clone(), rv=bn.running_var.clone())
    return out


def _saved_stats(y):
    """The batch mean / invstd the layer saved for its backward (ATen's native_batch_norm and ours save the same)."""
    fn = y.grad_fn
    if hasattr(fn, "_saved_result1"):  # ATen's batch_norm backward node: (output, save_mean, save_invstd, ...)
        return fn._saved_result1.clone(), fn._saved_result2.clone()
    _, _, mean, invstd = fn.saved_tensors
    return mean.clone(), invstd.clone()


def _bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}[t.dtype])


def _assert_same_bits(a, b):
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        diff = int((_bits(a[k]) != _bits(b[k])).sum())
        assert diff == 0, (k, diff, a[k].numel())


def _run(shape, dtype, seed=0, **kw):
    x, dy, ref = _inputs(shape, dtype, seed, **kw)
    mine = convert_batchnorm(copy.deepcopy(ref))
    assert type(mine) is BatchNorm2d
    a = _step(ref, x, dy)
    b = _step(mine, x, dy)
    assert b["y"].is_contiguous(memory_format=torch.channels_last) and b["dx"].is_contiguous(memory_format=torch.channels_last)
    _assert_same_bits(a, b)


@pytest.mark.parametrize("shape", RESNET50, ids=[f"M{s[0] * s[2] * s[3]}xC{s[1]}" for s in RESNET50])
def test_resnet50_shapes_bf16(shape):
    _run(shape, torch.bfloat16)


@pytest.mark.parametrize("shape", ODD, ids=lambda s: f"M{s[0] * s[2] * s[3]}xC{s[1]}")
def test_odd_shapes(shape):
    _run(shape, torch.bfloat16, seed=3)


def test_large_offset():
    _run((64, 64, 28, 28), torch.bfloat16, seed=5, offset=1000.0)


@pytest.mark.parametrize("kw", [{"momentum": 0.3}, {"track_running_stats": False}, {"eps": 1e-3}])
def test_layer_options(kw):
    _run((16, 64, 7, 7), torch.bfloat16, seed=9, **kw)


def test_non_finite_inputs_reach_the_outputs_as_in_aten():
    shape = (8, 32, 9, 9)
    x, dy, ref = _inputs(shape, torch.bfloat16, 7)
    x[0, 3, 0, 0] = float("nan")
    x[4, 9, 5, 2] = float("inf")
    x[2, 17, 1, 1] = -float("inf")
    dy[5, 21, 3, 3] = float("inf")
    dy[1, 30, 0, 8] = float("nan")
    mine = convert_batchnorm(copy.deepcopy(ref))
    a, b = _step(ref, x, dy), _step(mine, x, dy)
    for k in KEYS:
        assert torch.equal(torch.isfinite(a[k]), torch.isfinite(b[k])), k
    _assert_same_bits(a, b)  # a NaN result of the GPU's float arithmetic is the canonical NaN
    for c in (3, 9, 17):
        assert not torch.isfinite(b["y"][:, c]).any()
    for c in (21, 30):
        assert not torch.isfinite(b["dx"][:, c]).any() and not torch.isfinite(b["gb"][c])
    assert torch.isfinite(b["y"][:, 0]).all() and torch.isfinite(b["dx"][:, 0]).all()


def test_two_runs_are_bit_identical():
    shape = (64, 256, 28, 28)
    outs = []
    for _ in range(2):
        x, dy, ref = _inputs(shape, torch.bfloat16, 11)
        outs.append(_step(convert_batchnorm(ref), x, dy))
    _assert_same_bits(outs[0], outs[1])


def test_needs_input_grad_and_double_backward():
    x, dy, ref = _inputs((4, 16, 6, 6), torch.bfloat16, 13)
    bn = convert_batchnorm(ref)
    bn.weight.requires_grad_(False)
    xi = x.clone().requires_grad_()
    bn(xi).backward(dy)
    assert xi.grad is not None and bn.weight.grad is None and bn.bias.grad is not None
    xi = x.clone().requires_grad_()
    y = bn(xi)
    (g,) = torch.autograd.grad(y, xi, dy.clone().requires_grad_(), create_graph=True)
    with pytest.raises(RuntimeError, match="differentiate twice"):
        g.sum().backward()


def test_num_batches_tracked_and_eval_are_exact():
    x, dy, ref = _inputs((16, 64, 7, 7), torch.bfloat16, 17)
    ref.momentum = None
    mine = convert_batchnorm(copy.deepcopy(ref))
    for _ in range(3):
        _step(ref, x, dy)
        _step(mine, x, dy)
    assert torch.equal(ref.num_batches_tracked, mine.num_batches_tracked) and int(mine.num_batches_tracked) == 3
    ref.eval()
    mine.eval()
    with torch.no_grad():
        mine.running_mean.copy_(ref.running_mean)
        mine.running_var.copy_(ref.running_var)
        assert torch.equal(ref(x), mine(x))


def test_ineligible_inputs_stay_on_aten():
    x, dy, ref = _inputs((4, 16, 6, 6), torch.bfloat16, 19)
    mine = convert_batchnorm(copy.deepcopy(ref))
    for inp in (x.contiguous(), x.float(), x.half(), x[:, :, :, :5]):
        assert torch.equal(ref(inp), mine(inp))


def test_mini_ddp_convnet_step_under_bf16_autocast():
    from torchx_b200.ddp import Communicator, DistributedDataParallel

    def net():
        torch.manual_seed(0)
        return nn.Sequential(nn.Conv2d(3, 32, 3, padding=1, bias=False), nn.BatchNorm2d(32), nn.ReLU(), nn.Conv2d(32, 64, 3, stride=2, bias=False),
                             nn.BatchNorm2d(64), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(64, 10)).cuda().to(
                                 memory_format=torch.channels_last)

    g = torch.Generator(device="cuda").manual_seed(23)
    x = torch.randn(32, 3, 32, 32, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 10, (32,), device="cuda", generator=g)
    twin = net()
    (comm,) = Communicator.create_local([0], stage_mb=8)
    try:
        ddp = DistributedDataParallel(net(), comm)
        assert [type(m) for m in ddp.module if isinstance(m, nn.BatchNorm2d)] == [BatchNorm2d, BatchNorm2d]
        losses = []
        for model in (twin, ddp):
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    loss = nn.functional.cross_entropy(model(x), t)
                loss.backward()
                torch.cuda.synchronize()
            names = " ".join(e.name for e in prof.events())
            assert ("k_bn2d_norm" in names) == (model is ddp) and ("k_bn2d_bwd_elemt" in names) == (model is ddp)
            losses.append(loss.detach())
        comm.check()
        assert torch.equal(losses[0], losses[1])
        # at W = 1 the bf16-wire bucket pass leaves each gradient rounded to bf16
        for (n, p), q in zip(twin.named_parameters(), ddp.module.parameters()):
            assert torch.equal(p.grad.bfloat16().float(), q.grad), n
        assert ddp.copied_in_buckets == 0 and ddp.gathered_buckets > 0
    finally:
        comm.close()
