"""One rank of the native SyncBatchNorm checks (spawned by tests/test_syncbn_native_gpu.py) under init_pg("b200").

Every check runs the same work twice from the same state: as the package runs it (native kernels where the input allows,
fused ResNet blocks) and on the ATen-compute path the layer took before it had native kernels (``aten_path``: no input is
native-eligible and no block fuses, so SyncBatchNorm runs ``_FabricSyncBatchNorm`` over several ranks and ``F.batch_norm``
at one rank).  Results are compared bit for bit here; the worker saves the mismatching names, how many layers took the
native path, the op counter and, in the pair / groups modes, the results themselves.

--mode layers: single layers on ResNet-50's BatchNorm shapes with unequal per-rank batches, momentum None, no running
statistics, special values (+-0, NaN, +-inf, outputs that round to +-0), then one native forward + backward under
torch.cuda.set_sync_debug_mode("error").  At W = 1 the reference is F.batch_norm.
--mode mixed: ranks on different paths in one step (rank 0 NCHW, rank 1 an empty batch, rank 2 a misaligned view, the rest
native): single layers and a fused Bottleneck whose bn3 and downsample BatchNorm have the same width.
--mode frozen: a fused BasicBlock with a frozen conv1 and an input that needs no gradient, NCHW fp32 and channels-last bf16.
--mode nets: resnet50 and resnet18 converted to SyncBatchNorm, 3 SGD steps under the mini-DDP; the first fused step under
torch.profiler.
--mode pair / groups: small layers over a W = 2 world, and over two B200Groups of 2 in a W = 4 world."""
import argparse
import contextlib
import copy
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from torch import nn  # noqa: E402

import torchx_b200.nn.batchnorm as B  # noqa: E402
import torchx_b200.nn.resnet as R  # noqa: E402
from torchx_b200.nn import SyncBatchNorm  # noqa: E402

NATIVE = [0]  # layers that took the native path (native_eligible held in SyncBatchNorm)
_eligible = B.native_eligible


def _counting(bn, x):
    ok = _eligible(bn, x)
    NATIVE[0] += int(ok)
    return ok


B.native_eligible = _counting


@contextlib.contextmanager
def aten_path():
    """The path SyncBatchNorm took before its native kernels: no input is eligible and no ResNet block fuses."""
    saved = B.native_eligible, R._fusable
    B.native_eligible, R._fusable = (lambda bn, x: False), (lambda block, bns: False)
    try:
        yield
    finally:
        B.native_eligible, R._fusable = saved


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy()


# ResNet-50's BatchNorm shapes (C, H, W at 224 x 224)
R50 = [(64, 112, 112), (64, 56, 56), (256, 56, 56), (128, 56, 56), (128, 28, 28), (512, 28, 28), (256, 28, 28), (256, 14, 14),
       (1024, 14, 14), (512, 14, 14), (512, 7, 7), (2048, 7, 7)]
SIZES = [2, 3, 1, 2, 4, 1, 3, 2]


def layer_cases(world):
    cases = [(f"r50_{c}x{h}", (c, h, w), {}, None) for c, h, w in R50]
    cases += [("momentum_none", (64, 9, 9), {"momentum": None}, None),
              ("no_running_stats", (32, 6, 6), {"track_running_stats": False}, None),
              ("special", (64, 6, 6), {}, "special")]
    if world > 1:  # at one rank F.batch_norm refuses eps = 0
        cases.append(("eps_zero", (16, 5, 5), {"eps": 0.0}, "const"))
    return cases


def case_input(k, step, shape, n, special, device, rank):
    g = torch.Generator().manual_seed(10_000 * k + 100 * step + rank)
    C = shape[0]
    x = torch.randn((n,) + shape, generator=g) * 2 + torch.linspace(-3, 3, C).view(C, 1, 1)
    if special == "const" and n > 0:
        x[:, : C // 2] = 1.5  # zero variance: with eps = 0 torch's InvStd gives 0
    if special == "special" and n > 0:
        x[:, 0] = 0.0
        x[:, 1] = -0.0
        x[0, 2, 0, 0] = float("nan")
        x[0, 3, 0, 0] = float("inf")
        x[-1, 4, 0, 0] = float("-inf")
        x[:, 5] = 7.0  # constant: the output is the bias, some of which round to +-0 in bf16
    go = torch.randn((n,) + shape, generator=g)
    if special == "special" and n > 0:
        go[0, 6, 0, 0] = float("nan")
        go[:, 7] = -0.0
    cl = lambda t: t.to(device=device, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)  # noqa: E731
    return cl(x), cl(go)


def make_layer(shape, kw, special, device, group=None):
    torch.manual_seed(7)
    m = SyncBatchNorm(shape[0], process_group=group, **kw).to(device)
    with torch.no_grad():
        m.weight.uniform_(0.5, 1.5)
        m.bias.uniform_(-1, 1)
        if special == "special":
            m.bias[5::2] = 1e-42 * torch.sign(torch.randn(m.bias[5::2].shape))  # rounds to +-0 in bf16
            m.bias[6] = -1e-42
        if m.running_var is not None:
            m.running_var.uniform_(0.5, 2)
    return m


def run_layer(m, x, go):
    x = x.clone().requires_grad_()
    out = m(x)
    out.backward(go)
    got = {"out": bits(out), "grad_input": bits(x.grad if x.grad is not None else torch.zeros_like(x))}
    for n, p in (("grad_weight", m.weight.grad), ("grad_bias", m.bias.grad)):
        got[n] = bits(p) if p is not None else np.zeros(0, np.int32)
    m.weight.grad = m.bias.grad = None
    for n, b in m.named_buffers():
        got[n] = b.detach().cpu().numpy().copy()
    return got


def progress(*what):
    print(*what, flush=True)


def compare(tag, a, b, bad):
    for k in a:
        if a[k].shape != b[k].shape or a[k].tobytes() != b[k].tobytes():
            n = np.count_nonzero(a[k] != b[k]) if a[k].shape == b[k].shape else "shape"
            bad.append(f"{tag}.{k} ({n} of {a[k].size} differ)")
            progress("differs:", bad[-1])


def run_layers(rank, world, device, res, bad, cases, steps=2, group=None, sizes=SIZES, keep=False):
    for k, (name, shape, kw, special) in enumerate(cases):
        n = sizes[rank % len(sizes)]
        results = {}
        for impl in ("native", "aten"):
            m = make_layer(shape, kw, special, device, group)
            ctx = aten_path() if impl == "aten" else contextlib.nullcontext()
            results[impl] = []
            progress(name, impl)
            with ctx:
                for step in range(steps):
                    results[impl].append(run_layer(m, *case_input(k, step, shape, n, special, device, rank)))
        for step in range(steps):
            compare(f"{name}.{step}", results["native"][step], results["aten"][step], bad)
            if keep:
                for key, v in results["native"][step].items():
                    res[f"{name}.{step}.{key}"] = v


def run_nosync(rank, device, res):
    m = make_layer((64, 8, 8), {}, None, device)
    x, go = case_input(99, 0, (64, 8, 8), 2 + rank, None, device, rank)
    x.requires_grad_()
    before = NATIVE[0]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m(x).backward(go)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    res["nosync.native"] = np.array(NATIVE[0] - before)


def mixed_input(rank, n, shape, device, seed):
    g = torch.Generator().manual_seed(seed + rank)
    x = torch.randn((n,) + shape, generator=g).to(device=device, dtype=torch.bfloat16)
    if rank == 0:
        return x.contiguous()  # NCHW: ATen's compute
    x = x.contiguous(memory_format=torch.channels_last)
    if rank == 2:  # a channels-last view 2 bytes past a 16-byte boundary: ATen's compute
        buf = torch.empty(x.numel() + 8, dtype=torch.bfloat16, device=device)
        v = buf[1:1 + x.numel()].view(n, shape[1], shape[2], shape[0]).permute(0, 3, 1, 2)
        v.copy_(x)
        assert v.is_contiguous(memory_format=torch.channels_last) and v.data_ptr() % 16 != 0
        return v
    return x


def run_mixed(rank, world, device, res, bad):
    from torchvision.models.resnet import Bottleneck

    sizes = [3, 0, 2] + [2 + r % 2 for r in range(3, world)]  # rank 1 has an empty batch
    n = sizes[rank]
    # two layers of one width back to back, then a fused Bottleneck whose bn3 and downsample BatchNorm are both 64 wide
    for k, shape in enumerate([(64, 10, 10), (16, 7, 7)]):
        x = mixed_input(rank, n, shape, device, 100 * k)
        go = mixed_input(rank, n, shape, device, 100 * k + 50)
        got = {}
        for impl in ("native", "aten"):
            progress("layers", k, impl)
            ms = [make_layer(shape, {}, None, device) for _ in range(2)]
            with aten_path() if impl == "aten" else contextlib.nullcontext():
                xi = x.clone().requires_grad_()
                out = ms[1](ms[0](xi))
                out.backward(go)
            got[impl] = {"out": bits(out), "grad_input": bits(xi.grad if xi.grad is not None else torch.zeros_like(xi))}
            for j, m in enumerate(ms):
                for name, b in m.named_buffers():
                    got[impl][f"{j}.{name}"] = b.cpu().numpy()
                if n > 0:
                    got[impl][f"{j}.grad_weight"] = bits(m.weight.grad)
        compare(f"layers{k}", got["native"], got["aten"], bad)

    torch.manual_seed(3)
    base = Bottleneck(64, 16, downsample=nn.Sequential(nn.Conv2d(64, 64, 1, bias=False), nn.BatchNorm2d(64)))
    base = SyncBatchNorm.convert_sync_batchnorm(base).to(device)
    with torch.no_grad():
        for m in base.modules():
            if isinstance(m, SyncBatchNorm):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.5, 0.5)
    base.train()
    if rank != 0:
        base = base.to(memory_format=torch.channels_last)
    x = mixed_input(rank, n, (64, 8, 8), device, 7)
    go = mixed_input(rank, n, (64, 8, 8), device, 8)
    got = {}
    for impl in ("native", "aten"):
        blk = R.fuse_resnet(copy.deepcopy(base))
        assert type(blk).__name__ == "FusedBottleneck"
        with aten_path() if impl == "aten" else contextlib.nullcontext():
            for step in range(2):
                progress("bottleneck", impl, step)
                xi = x.clone().requires_grad_()
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    out = blk(xi)
                out.backward(go)
                got[impl] = got.get(impl, {})
                got[impl][f"{step}.out"] = bits(out)
                got[impl][f"{step}.grad_input"] = bits(xi.grad if xi.grad is not None else torch.zeros_like(xi))
        for name, p in blk.named_parameters():
            if p.grad is not None:
                got[impl][f"grad.{name}"] = bits(p.grad)
        for name, b in blk.named_buffers():
            got[impl][name] = b.cpu().numpy()
    compare("bottleneck", got["native"], got["aten"], bad)


def run_frozen(rank, world, device, res, bad):
    """A fused BasicBlock whose conv1 is frozen, fed an input that needs no gradient: bn1's input needs none while its
    weight and bias are trainable, so its backward forms no dx and runs no allreduce.  NCHW fp32 (ATen's compute inside
    the fused block) and channels-last bf16 under autocast (the native kernels)."""
    from torchvision.models.resnet import BasicBlock

    for tag, bf16 in (("nchw_fp32", False), ("channels_last_bf16", True)):
        torch.manual_seed(4)
        base = SyncBatchNorm.convert_sync_batchnorm(BasicBlock(16, 16)).to(device)
        base.conv1.weight.requires_grad_(False)
        fmt = torch.channels_last if bf16 else torch.contiguous_format
        base = base.to(memory_format=fmt).train()
        g = torch.Generator().manual_seed(20 + rank)
        x = torch.randn(2 + rank, 16, 8, 8, generator=g).to(device).contiguous(memory_format=fmt)
        go = torch.randn(2 + rank, 16, 8, 8, generator=g).to(device).contiguous(memory_format=fmt)
        got = {}
        for impl in ("native", "aten"):
            progress("frozen", tag, impl)
            blk = R.fuse_resnet(copy.deepcopy(base))
            with aten_path() if impl == "aten" else contextlib.nullcontext():
                for step in range(2):
                    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
                        out = blk(x)
                    out.backward(go.to(out.dtype))
                    got.setdefault(impl, {})[f"{step}.out"] = bits(out)
            for name, p in blk.named_parameters():
                got[impl][f"grad.{name}"] = bits(p.grad) if p.grad is not None else np.zeros(0, np.int32)
            for name, b in blk.named_buffers():
                got[impl][name] = b.cpu().numpy()
        compare(tag, got["native"], got["aten"], bad)


def run_nets(rank, world, device, res, bad, comm):
    import torchvision

    from torchx_b200.ddp import DistributedDataParallel

    torch.use_deterministic_algorithms(True)
    torch.backends.cudnn.benchmark = False
    names = {}
    for arch in ("resnet50", "resnet18"):
        torch.manual_seed(0)
        base = SyncBatchNorm.convert_sync_batchnorm(torchvision.models.__dict__[arch]())
        base = base.to(device).to(memory_format=torch.channels_last)
        g = torch.Generator().manual_seed(5 + rank)
        x = torch.randn(4, 3, 64, 64, generator=g).to(device).contiguous(memory_format=torch.channels_last)
        t = torch.randint(0, 1000, (4,), generator=g).to(device)
        got = {}
        for impl in ("native", "aten"):
            net = copy.deepcopy(base)
            model = DistributedDataParallel(net, comm=comm)
            opt = torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9)
            losses = []
            with aten_path() if impl == "aten" else contextlib.nullcontext():
                for step in range(3):
                    opt.zero_grad(set_to_none=True)

                    def fwd_bwd():
                        with torch.autocast("cuda", dtype=torch.bfloat16):
                            loss = F.cross_entropy(model(x), t)
                        loss.backward()
                        return loss.detach()

                    if step == 0 and impl == "native":
                        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                            loss = fwd_bwd()
                            torch.cuda.synchronize()
                        names[arch] = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                    else:
                        loss = fwd_bwd()
                    losses.append(bits(loss))
                    opt.step()
            torch.cuda.synchronize()
            got[impl] = {f"loss{i}": v for i, v in enumerate(losses)}
            for n, p in net.named_parameters():
                got[impl][n] = bits(p)
                got[impl]["grad." + n] = bits(p.grad)
            for n, b in net.named_buffers():
                got[impl][n] = b.cpu().numpy()
            del model
        compare(arch, got["native"], got["aten"], bad)
        k = names[arch]
        res[f"{arch}.kernels.aten_bn"] = np.array(sum(1 for n in k if re.search(r"batch_norm", n)))
        res[f"{arch}.kernels.relu"] = np.array(sum(1 for n in k if re.search(r"clamp_min|clamp_scalar", n)))
        res[f"{arch}.kernels.threshold"] = np.array(sum(1 for n in k if re.search(r"threshold", n)))
        res[f"{arch}.kernels.native_bn"] = np.array(sum(1 for n in k if re.search(r"k_bn2d_", n)))


PAIR_CASES = [("pair_a", (64, 6, 6), {}, None), ("pair_b", (32, 5, 5), {"momentum": None}, None)]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--device", type=int, required=True)
    ap.add_argument("--shm", required=True)
    ap.add_argument("--mode", choices=("layers", "mixed", "frozen", "nets", "pair", "groups"), required=True)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    os.environ.update(RANK=str(a.rank), WORLD_SIZE=str(a.world), LOCAL_RANK=str(a.rank), B2_DEVICE=str(a.device),
                      B2_SHM_NAME=a.shm)

    import torchx_b200.distributed as D

    device = D.init_pg("b200", stage_mb=8, timeout_s=120)
    comm = D.communicator()
    comm.set_timeout(60.0)
    comm.set_max_ctas(8)
    rank, world = D.rank(), D.world_size()
    res, bad = {}, []
    if a.mode == "layers":
        run_layers(rank, world, device, res, bad, layer_cases(world))
        run_nosync(rank, device, res)
    elif a.mode == "mixed":
        run_mixed(rank, world, device, res, bad)
    elif a.mode == "frozen":
        run_frozen(rank, world, device, res, bad)
    elif a.mode == "nets":
        run_nets(rank, world, device, res, bad, comm)
    elif a.mode == "pair":
        run_layers(rank, world, device, res, bad, PAIR_CASES, keep=True)
    else:
        groups = [D.new_group([0, 1]), D.new_group([2, 3])]
        mine = groups[rank // 2]
        run_layers(rank % 2, 2, device, res, bad, PAIR_CASES, group=mine, keep=True)
    torch.cuda.synchronize()
    comm.check()
    res["native"] = np.array(NATIVE[0])
    res["bad"] = np.array("\n".join(bad))
    res["op_count"] = np.array(comm.op_count)
    np.savez(a.out, **res)
    D.barrier()
    comm.close()
    print(f"rank {a.rank} ok", flush=True)


if __name__ == "__main__":
    main()
