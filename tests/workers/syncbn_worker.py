"""One rank of the SyncBatchNorm checks (spawned by tests/test_syncbn_gpu.py) under init_pg("b200"), no process group.

--mode module: torchx_b200.nn.SyncBatchNorm forward + backward on several layouts and dtypes, next to a single-process
reference that every rank computes for itself from the same seeds: torch's SyncBatchNorm code path with its all_gather
replaced by an exact concatenation and its allreduce by the rank-order fp32 sum.  Also runs one forward + backward under
torch.cuda.set_sync_debug_mode("error").
--mode ddp: a small conv net converted with convert_sync_batchnorm, trained a few steps under the mini-DDP with buckets
small enough to fire while SyncBatchNorm's backward collectives are still being issued; then the same training without
overlap (gradients averaged after backward, every collective on the current stream).
--mode torch: torch.nn.SyncBatchNorm itself under a torch.distributed group (--backend gloo with every rank on one GPU, or
nccl with one GPU per rank): single layers over several steps (momentum None, no running statistics, no affine, empty ranks,
bf16 autocast, eval) and a converted conv net trained with torch's recipe; then the same under init_pg("b200") with this
package's SyncBatchNorm and the mini-DDP."""
import argparse
import copy
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from torch import nn  # noqa: E402

# name, dtype, channels_last, per-rank shape after the batch dimension, per-rank batch sizes (cut to the world size)
CASES = [
    ("fp32_nchw", torch.float32, False, (6, 5, 4), [4, 7, 1, 3]),
    ("fp32_nchw_empty_rank", torch.float32, False, (6, 5, 4), [5, 0, 3, 0]),
    ("fp32_channels_last", torch.float32, True, (16, 3, 3), [2, 5, 4, 1]),
    ("fp32_nc", torch.float32, False, (33,), [9, 2, 17, 5]),
    ("fp32_nc_empty_rank", torch.float32, False, (33,), [0, 6, 1, 8]),
    ("bf16_autocast_channels_last", torch.bfloat16, True, (8, 4, 4), [3, 6, 0, 2]),
    ("bf16_autocast_nc", torch.bfloat16, False, (24,), [7, 1, 4, 4]),
]
EPS, MOMENTUM = 1e-5, 0.1


def bits(t: torch.Tensor) -> np.ndarray:
    t = t.detach().contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy()


def case_data(k, dtype, channels_last, shape, sizes, device):
    g = torch.Generator().manual_seed(1000 + k)
    C = shape[0]
    xs = [(torch.randn((n,) + shape, generator=g) * 2 + torch.linspace(-1, 1, C).view((C,) + (1,) * (len(shape) - 1)))
          for n in sizes]
    gos = [torch.randn((n,) + shape, generator=g) for n in sizes]
    w, b = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    rm, rv = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    xs = [x.to(device=device, dtype=dtype).contiguous(memory_format=fmt) for x in xs]
    gos = [x.to(device=device, dtype=dtype).contiguous(memory_format=fmt) for x in gos]
    return xs, gos, w.to(device), b.to(device), rm.to(device), rv.to(device)


def reference(xs, gos, w, b, rm, rv):
    """torch's SyncBatchNorm function (torch/nn/modules/_functions.py) for every rank at once: exact concatenation for the
    all_gather, the rank-order fp32 sum for the allreduce.  Returns per rank (out, grad_input, running_mean, running_var)."""
    C = xs[0].shape[1]
    rows = []
    for x in xs:
        if x.numel() > 0:
            mean, invstd = torch.batch_norm_stats(x, EPS)
            rows.append(torch.cat([mean, invstd, torch.full((1,), x.numel() // C, dtype=mean.dtype, device=x.device)]))
        else:
            rows.append(torch.zeros(2 * C + 1, dtype=torch.float32, device=x.device))
    combined = torch.stack(rows)
    mean_all, invstd_all, count_all = torch.split(combined, C, dim=1)
    mask = count_all.squeeze(-1) >= 1
    count_all, mean_all, invstd_all = count_all[mask], mean_all[mask], invstd_all[mask]
    counts = count_all.view(-1)
    res, sums = [], []
    for x, go in zip(xs, gos):
        rm_r, rv_r = rm.clone(), rv.clone()
        mean, invstd = torch.batch_norm_gather_stats_with_counts(x, mean_all, invstd_all, rm_r, rv_r, MOMENTUM, EPS, counts)
        out = torch.batch_norm_elemt(x, w, b, mean, invstd, EPS) if x.numel() > 0 else torch.empty_like(x)
        if x.numel() > 0:
            sum_dy, sum_dy_xmu, _, _ = torch.batch_norm_backward_reduce(go, x, mean, invstd, w, True, True, True)
            sums.append(torch.cat([sum_dy, sum_dy_xmu]))
        else:
            sums.append(torch.zeros(2 * C, dtype=torch.float32, device=x.device))
        res.append([out, None, rm_r, rv_r, mean, invstd])
    total = sums[0].clone()
    for s in sums[1:]:
        total = total + s
    sum_dy, sum_dy_xmu = torch.split(total, C)
    for x, go, r in zip(xs, gos, res):
        if x.numel() > 0:
            r[1] = torch.batch_norm_backward_elemt(go, x, r[4], r[5], w, sum_dy, sum_dy_xmu, count_all.to(torch.int32))
        else:
            r[1] = torch.zeros_like(x)
    return [r[:4] for r in res]


def run_module(comm, rank, world, device, res):
    from torchx_b200.nn import SyncBatchNorm

    for k, (name, dtype, cl, shape, sizes) in enumerate(CASES):
        sizes = sizes[:world]
        xs, gos, w, b, rm, rv = case_data(k, dtype, cl, shape, sizes, device)
        m = SyncBatchNorm(shape[0], eps=EPS, momentum=MOMENTUM).to(device)
        with torch.no_grad():
            m.weight.copy_(w)
            m.bias.copy_(b)
            m.running_mean.copy_(rm)
            m.running_var.copy_(rv)
        x = xs[rank].clone().requires_grad_()
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype == torch.bfloat16):
            out = m(x)
        out.backward(gos[rank])
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype == torch.bfloat16):
            want = reference(xs, gos, w, b, rm, rv)[rank]
        grad = x.grad if x.grad is not None else torch.zeros_like(x)
        for tag, g, wv in (("out", out, want[0]), ("grad", grad, want[1]), ("rm", m.running_mean, want[2]),
                           ("rv", m.running_var, want[3])):
            res[f"{name}.{tag}.got"] = bits(g)
            res[f"{name}.{tag}.want"] = bits(wv)
        assert out.dtype == want[0].dtype and out.stride() == want[0].stride(), name

    # no device-to-host sync anywhere in a fabric forward + backward
    m = SyncBatchNorm(4).to(device)
    x = torch.randn(3 + rank, 4, 5, device=device, requires_grad=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m(x).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    res["nosync.ok"] = np.array(1)


def make_net():
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3, bias=False), nn.BatchNorm2d(8), nn.ReLU(), nn.Conv2d(8, 16, 3, bias=False),
                         nn.BatchNorm2d(16), nn.ReLU(), nn.Conv2d(16, 16, 1), nn.BatchNorm2d(16), nn.ReLU(),
                         nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(16, 5), nn.BatchNorm1d(5))


def batches(rank, steps, device):
    for s in range(steps):
        g = torch.Generator().manual_seed(100 * s + rank)
        n = 3 + (rank + s) % 3
        yield torch.randn(n, 3, 9, 9, generator=g).to(device), torch.randint(0, 5, (n,), generator=g).to(device)


def run_ddp(comm, rank, world, device, res, steps=4):
    from torchx_b200.ddp import DistributedDataParallel
    from torchx_b200.nn import SyncBatchNorm

    net = SyncBatchNorm.convert_sync_batchnorm(make_net()).to(device)
    ref = copy.deepcopy(net)
    model = DistributedDataParallel(net, comm=comm, bucket_cap_mb=1 / 4096, first_bucket_mb=1 / 4096, wire="f32")
    assert len(model.buckets) >= 4 and comm.ordered_stream is model._comm_stream
    opt = torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9)
    for x, y in batches(rank, steps, device):
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(model(x), y).backward()
        opt.step()
    torch.cuda.synchronize()
    comm.check()

    # the same training with no overlap: every collective on the current stream, gradients averaged after backward
    saved, comm.ordered_stream = comm.ordered_stream, None
    ropt = torch.optim.SGD(ref.parameters(), lr=0.1, momentum=0.9)
    for x, y in batches(rank, steps, device):
        ropt.zero_grad(set_to_none=True)
        F.cross_entropy(ref(x), y).backward()
        for p in ref.parameters():
            comm.allreduce_(p.grad, scale=1.0 / world, wire="f32")
        ropt.step()
    comm.ordered_stream = saved
    torch.cuda.synchronize()
    comm.check()
    for (k, v), (k2, v2) in zip(net.state_dict().items(), ref.state_dict().items()):
        assert k == k2
        res[f"ddp.{k}"] = v.detach().cpu().numpy()
        res[f"ref.{k}"] = v2.detach().cpu().numpy()


# torch mode: torch.nn.SyncBatchNorm over a torch.distributed group, then torchx_b200.nn.SyncBatchNorm on the fabric, on the
# same inputs.  name, module kwargs, dtype, channels_last, shape after the batch dimension, batch sizes (cycled over ranks)
TORCH_CASES = [
    ("default", {}, torch.float32, False, (6, 5, 4), [4, 7, 1, 3]),
    ("momentum_none", {"momentum": None}, torch.float32, True, (16, 3, 3), [2, 5, 4, 1]),
    ("no_running_stats", {"track_running_stats": False}, torch.float32, False, (33,), [9, 2, 17, 5]),
    ("no_affine_empty_rank", {"affine": False, "eps": 1e-3, "momentum": 0.3}, torch.float32, False, (6, 5, 4), [5, 0, 3, 0]),
    ("bf16_autocast", {}, torch.bfloat16, True, (8, 4, 4), [3, 6, 2, 2]),
]
TORCH_STEPS = 3


def run_layers(cls, rank, world, device, res, prefix):
    """Every TORCH_CASES layer for TORCH_STEPS training steps and one eval forward: outputs, input / weight / bias gradients,
    running statistics and num_batches_tracked after each step."""
    for k, (name, kw, dtype, cl, shape, sizes) in enumerate(TORCH_CASES):
        sizes = [sizes[r % len(sizes)] for r in range(world)]
        torch.manual_seed(7)
        m = cls(shape[0], **kw).to(device)
        if m.affine:
            with torch.no_grad():
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-1, 1)
        for step in range(TORCH_STEPS + 1):
            xs, gos, _, _, _, _ = case_data(100 * k + step, dtype, cl, shape, sizes, device)
            m.train(step < TORCH_STEPS)
            x = xs[rank].clone().requires_grad_()
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype == torch.bfloat16):
                out = m(x)
            key = f"{prefix}.{name}.{step}"
            res[f"{key}.out"] = bits(out)
            if step == TORCH_STEPS:
                continue
            if m.affine:
                m.weight.grad = m.bias.grad = None
            out.backward(gos[rank])
            res[f"{key}.grad_input"] = bits(x.grad if x.grad is not None else torch.zeros_like(x))
            if m.affine:
                res[f"{key}.grad_weight"] = bits(m.weight.grad)
                res[f"{key}.grad_bias"] = bits(m.bias.grad)
            for b, v in m.named_buffers():
                res[f"{key}.{b}"] = v.detach().cpu().numpy()


def train_torch_recipe(net, rank, world, device, steps=4):
    """torch's recipe: gradients summed with dist.all_reduce and scaled by 1 / W after backward."""
    import torch.distributed as dist

    opt = torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9)
    for x, y in batches(rank, steps, device):
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(net(x), y).backward()
        for p in net.parameters():
            dist.all_reduce(p.grad)
            p.grad.mul_(1.0 / world)
        opt.step()


def run_torch(a, res):
    """torch.nn.SyncBatchNorm under a real process group, then this package's SyncBatchNorm under init_pg("b200")."""
    import torch.distributed as dist

    import torchx_b200.distributed as D
    from torchx_b200.ddp import DistributedDataParallel
    from torchx_b200.nn import SyncBatchNorm

    device = torch.device("cuda", a.device)
    torch.cuda.set_device(device)
    dist.init_process_group(a.backend, init_method=f"tcp://127.0.0.1:{a.port}", rank=a.rank, world_size=a.world)
    run_layers(nn.SyncBatchNorm, a.rank, a.world, device, res, "torch")
    net = nn.SyncBatchNorm.convert_sync_batchnorm(make_net()).to(device)
    train_torch_recipe(net, a.rank, a.world, device)
    for k, v in net.state_dict().items():
        res[f"torch.train.{k}"] = v.detach().cpu().numpy()
    torch.cuda.synchronize()
    dist.destroy_process_group()

    D.init_pg("b200", stage_mb=8, timeout_s=60)
    comm = D.communicator()
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    assert not dist.is_initialized() and D._on_fabric()
    run_layers(SyncBatchNorm, a.rank, a.world, device, res, "fabric")
    net = SyncBatchNorm.convert_sync_batchnorm(make_net()).to(device)
    model = DistributedDataParallel(net, comm=comm, bucket_cap_mb=1 / 4096, first_bucket_mb=1 / 4096, wire="f32")
    opt = torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9)
    for x, y in batches(a.rank, 4, device):
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(model(x), y).backward()
        opt.step()
    for k, v in net.state_dict().items():
        res[f"fabric.train.{k}"] = v.detach().cpu().numpy()
    return comm


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--device", type=int, required=True)
    ap.add_argument("--shm", required=True)
    ap.add_argument("--mode", choices=("module", "ddp", "torch"), required=True)
    ap.add_argument("--backend", default="nccl", help="torch mode: the process group torch's SyncBatchNorm runs on")
    ap.add_argument("--port", type=int, default=0, help="torch mode: the process group's TCP port")
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    os.environ.update(RANK=str(a.rank), WORLD_SIZE=str(a.world), LOCAL_RANK=str(a.rank), B2_DEVICE=str(a.device),
                      B2_SHM_NAME=a.shm)

    import torch.distributed as dist

    import torchx_b200.distributed as D

    res = {}
    if a.mode == "torch":
        comm = run_torch(a, res)
    else:
        device = D.init_pg("b200", stage_mb=8, timeout_s=60)
        comm = D.communicator()
        comm.set_timeout(30.0)
        comm.set_max_ctas(8)
        assert not dist.is_initialized() and D._on_fabric()
        (run_module if a.mode == "module" else run_ddp)(comm, D.rank(), D.world_size(), device, res)
    torch.cuda.synchronize()
    comm.check()
    np.savez(a.out, **res)
    D.barrier()
    comm.close()
    print(f"rank {a.rank} ok", flush=True)


if __name__ == "__main__":
    main()
