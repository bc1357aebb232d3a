"""ReLU and the residual add inside the native BatchNorm passes (torchx_b200.nn.resnet) on the GPU: each fused layer, and
whole torchvision ResNets over SGD steps, give the bits of the unfused native BatchNorm followed by ATen's add_ and relu_;
the fused step launches no ATen ReLU kernel; hooks, eval mode and fp16 take the unfused path; a captured CUDA graph of
a fused step replays to the eager bits."""
import copy
import os
import re

import pytest
import torch
from torch import nn

from torchx_b200.nn import BatchNorm2d, convert_batchnorm, fuse_resnet

torchvision = pytest.importorskip("torchvision")
pytestmark = pytest.mark.gpu

# (N, C, H, W) of the 12 distinct [M, C] shapes of ResNet-50's 49 fused layers at B = 256; the last four are the bn3 layers
# that add the residual
RESNET50 = [(256, 64, 112, 112), (256, 64, 56, 56), (256, 128, 56, 56), (256, 128, 28, 28), (256, 256, 28, 28), (256, 256, 14, 14),
            (256, 512, 14, 14), (256, 512, 7, 7), (256, 256, 56, 56), (256, 512, 28, 28), (256, 1024, 14, 14), (256, 2048, 7, 7)]
ODD = [(2, 8, 1, 1), (3, 24, 1, 1), (7, 72, 1, 1), (5, 8, 13, 193), (5, 72, 13, 193), (1, 2056, 3, 5)]


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _inputs(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = shape[1]
    x = _cl(torch.randn(shape, device="cuda", generator=g).bfloat16())
    r = _cl(torch.randn(shape, device="cuda", generator=g).bfloat16())
    dz = _cl(torch.randn(shape, device="cuda", generator=g).bfloat16())
    bn = convert_batchnorm(nn.BatchNorm2d(c).cuda())
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5, generator=g)
        bn.bias.uniform_(-0.5, 0.5, generator=g)
        bn.running_mean.uniform_(-1.0, 1.0, generator=g)
        bn.running_var.uniform_(0.5, 2.0, generator=g)
    return x, r, dz, bn


def _unfused(bn, x, r, dz):
    xi = x.clone().requires_grad_()
    ri = r.clone().requires_grad_() if r is not None else None
    y = bn(xi)
    _, _, mean, invstd = y.grad_fn.saved_tensors
    if ri is not None:
        y += ri
    z = torch.relu_(y)
    z.backward(dz)
    return _result(bn, z, xi, ri, mean, invstd)


def _fused(bn, x, r, dz):
    xi = x.clone().requires_grad_()
    ri = r.clone().requires_grad_() if r is not None else None
    _, mean, _, invstd, _ = stats = bn.batch_stats(xi)
    z = bn.normalise(stats, ri, relu=True)
    z.backward(dz)
    return _result(bn, z, xi, ri, mean, invstd)


def _result(bn, z, xi, ri, mean, invstd):
    out = {"z": z.detach(), "dx": xi.grad, "gw": bn.weight.grad.clone(), "gb": bn.bias.grad.clone(), "mean": mean.clone(),
           "invstd": invstd.clone(), "rm": bn.running_mean.clone(), "rv": bn.running_var.clone()}
    if ri is not None:
        out["dr"] = ri.grad
    return out


def _bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}[t.dtype])


def _assert_same_bits(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        diff = int((_bits(a[k]) != _bits(b[k])).sum())
        assert diff == 0, (k, diff, a[k].numel())


def _compare(x, r, dz, bn):
    ref = copy.deepcopy(bn)
    a = _unfused(ref, x, r, dz)
    b = _fused(bn, x, r, dz)
    assert b["z"].is_contiguous(memory_format=torch.channels_last) and b["dx"].is_contiguous(memory_format=torch.channels_last)
    _assert_same_bits(a, b)


@pytest.mark.parametrize("residual", [False, True], ids=["relu", "add_relu"])
@pytest.mark.parametrize("shape", RESNET50 + ODD, ids=[f"M{s[0] * s[2] * s[3]}xC{s[1]}" for s in RESNET50 + ODD])
def test_layer_bits(shape, residual):
    x, r, dz, bn = _inputs(shape, 1)
    _compare(x, r if residual else None, dz, bn)


@pytest.mark.parametrize("residual", [False, True], ids=["relu", "add_relu"])
@pytest.mark.parametrize("shape", [(256, 2048, 7, 7), (5, 72, 13, 193)], ids=["M12544xC2048", "M12545xC72"])
def test_gradient_in_another_layout(shape, residual):
    """An NCHW-contiguous dz, as a mean's backward gives ResNet's last block: the fused reduce masks it in place."""
    x, r, dz, bn = _inputs(shape, 4)
    dz = dz.contiguous()
    assert not dz.is_contiguous(memory_format=torch.channels_last)
    _compare(x, r if residual else None, dz, bn)


@pytest.mark.parametrize("residual", [False, True], ids=["relu", "add_relu"])
def test_special_values(residual):
    """±0, NaN and ±inf in x, the residual and dz, and BatchNorm outputs that round to ±0 in bf16 (channel 3: a weight of
    1e-42 and no bias), where the fused ReLU must give the sign of zero ATen's relu_ gives."""
    shape = (4, 16, 5, 7)
    x, r, dz, bn = _inputs(shape, 2)
    special = torch.tensor([0.0, -0.0, float("nan"), float("inf"), -float("inf")], device="cuda").bfloat16()
    with torch.no_grad():
        x[0, 1, 0, :5] = special          # channel 1: NaN and inf statistics
        x[1, 2, 1, 0] = float("inf")      # channel 2: inf
        for i in range(5):                # scattered special residuals and gradients
            r[i % 4, 4 + i, 2, 3] = special[i]
            r[(i + 1) % 4, 5, i, 1] = special[i]
            dz[i % 4, 6 + i, 3, 2] = special[i]
            dz[(i + 2) % 4, 3, i, 4] = special[i]
        bn.weight[3] = 1e-42
        bn.bias[3] = 0.0
        r[:, 3] = torch.where(torch.arange(7, device="cuda") % 2 == 0, 0.0, -0.0).bfloat16()  # ±0 + ±0
        r[0, 8] = -bn(x)[0, 8]  # exact cancellation, y + (-y); the call's running-statistics update is undone below
        bn.running_mean.zero_()
        bn.running_var.fill_(1.0)
        bn.num_batches_tracked.zero_()
    _compare(x, r if residual else None, dz, bn)


def _model(name):
    torch.manual_seed(0)
    return getattr(torchvision.models, name)().cuda().to(memory_format=torch.channels_last)


def _batch(n, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = _cl(torch.randn(n, 3, 224, 224, device="cuda", generator=g))
    return x, torch.randint(0, 1000, (n,), device="cuda", generator=g)


class _Deterministic:
    def __enter__(self):
        os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
        self.det, self.bench = torch.are_deterministic_algorithms_enabled(), torch.backends.cudnn.benchmark
        torch.use_deterministic_algorithms(True)
        torch.backends.cudnn.benchmark = False

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.det)
        torch.backends.cudnn.benchmark = self.bench


def _kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


RELU = r"clamp_min|clamp_scalar"  # relu_ is clamp_min_(0): its kernel is launch_clamp_scalar's


def _count(names, pattern):
    return sum(1 for n in names if re.search(pattern, n))


def _train(model, x, t, steps, profile_first=False, dtype=torch.bfloat16):
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9)
    losses, names = [], None

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=dtype):
            loss = nn.functional.cross_entropy(model(x), t)
        loss.backward()
        return loss.detach()

    for i in range(steps):
        if i == 0 and profile_first:
            loss, names = _kernels(step)
        else:
            loss = step()
        losses.append(loss)
        opt.step()
    return losses, names


def _assert_models_equal(a, b, losses_a, losses_b):
    assert [_bits(l).item() for l in losses_a] == [_bits(l).item() for l in losses_b]
    for (n, p), q in zip(a.named_parameters(), b.parameters()):
        assert torch.equal(_bits(p.detach()), _bits(q.detach())), n
        assert torch.equal(_bits(p.grad), _bits(q.grad)), n
    for (n, p), q in zip(a.named_buffers(), b.buffers()):
        assert torch.equal(p, q), n


@pytest.mark.parametrize("name", ["resnet50", "resnet18"])
def test_whole_model_bits(name):
    base = _model(name)
    plain = convert_batchnorm(copy.deepcopy(base))
    fused = fuse_resnet(convert_batchnorm(copy.deepcopy(base)))
    x, t = _batch(8)
    with _Deterministic():
        la, names_a = _train(plain, x, t, 3, profile_first=True)
        lb, names_b = _train(fused, x, t, 3, profile_first=True)
    _assert_models_equal(plain, fused, la, lb)
    assert _count(names_a, RELU) > 0 and _count(names_a, r"threshold") > 0
    assert _count(names_b, RELU) == 0 and _count(names_b, r"threshold") == 0
    blocks = sum(1 for m in base.modules() if isinstance(m, (torchvision.models.resnet.Bottleneck, torchvision.models.resnet.BasicBlock)))
    add = r"CUDAFunctor_add|AddFunctor"
    assert _count(names_a, add) - _count(names_b, add) == blocks


@pytest.mark.parametrize("case", ["hook", "eval", "fp16"])
def test_fallback_bits(case, monkeypatch):
    base = _model("resnet18")
    plain = convert_batchnorm(copy.deepcopy(base))
    fused = fuse_resnet(convert_batchnorm(copy.deepcopy(base)))
    x, t = _batch(4)
    fused_layers = []  # every layer that takes the fused path starts with BatchNorm2d.batch_stats
    batch_stats = BatchNorm2d.batch_stats
    monkeypatch.setattr(BatchNorm2d, "batch_stats", lambda bn, inp: fused_layers.append(bn) or batch_stats(bn, inp))
    with _Deterministic():
        if case == "eval":
            plain.eval()
            fused.eval()
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                a = plain(x)
                b = fused(x)
            assert torch.equal(_bits(a), _bits(b))
        else:
            if case == "hook":
                seen = []
                for m in (plain, fused):
                    m.layer1[0].bn2.register_forward_hook(lambda mod, i, o: seen.append(o.shape))
            dtype = torch.float16 if case == "fp16" else torch.bfloat16
            la, _ = _train(plain, x, t, 2, dtype=dtype)
            lb, _ = _train(fused, x, t, 2, dtype=dtype)
            _assert_models_equal(plain, fused, la, lb)
            if case == "hook":
                assert len(seen) == 4
    # nothing fused in eval and fp16; with the hook, all but the hooked block's two layers, in both steps
    hooked = {id(fused.layer1[0].bn1), id(fused.layer1[0].bn2)}
    assert len(fused_layers) == (2 * 15 if case == "hook" else 0)
    assert not hooked & {id(bn) for bn in fused_layers}


def test_graph_replay_bits():
    """A captured forward + backward of a fused resnet18 replays to what the same step computes eagerly."""
    base = fuse_resnet(convert_batchnorm(_model("resnet18")))
    x, t = _batch(8)

    def step(model):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = nn.functional.cross_entropy(model(x), t)
        loss.backward()
        return loss

    with _Deterministic():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                step(base)
        torch.cuda.current_stream().wait_stream(side)
        eager = copy.deepcopy(base)
        for m in (base, eager):
            for p in m.parameters():
                p.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_loss = step(base)
        graph.replay()
        loss = step(eager)
        torch.cuda.synchronize()
    assert any(type(m) is BatchNorm2d for m in base.modules())
    _assert_models_equal(eager, base, [loss.detach()], [static_loss.detach()])
