"""An unmodified-torch training script on the H100 fabric: ``dist.init_process_group("b200")``.

    python -m torchx_b200.cli.main run -s local_cuda dist.ddp -j 1x2 --script examples/train_stock_ddp.py -- --steps 20

Everything below is stock torch - ``torch.nn.SyncBatchNorm.convert_sync_batchnorm``, ``DistributedDataParallel`` and its
own ``bf16_compress_hook`` - except the import that registers the ``"b200"`` backend.  Every collective (DDP's
construction broadcast, bucket allreduces, buffer broadcasts, SyncBatchNorm's exchanges) runs on the native communicator;
no gloo or NCCL group is created.  At the end every rank prints a hash of its parameters; they must agree.
"""
import argparse
import hashlib
import os
import sys

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.distributed.algorithms.ddp_comm_hooks import default_hooks

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchx_b200.distributed  # noqa: E402,F401  (registers the "b200" backend)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()

    dist.init_process_group("b200")
    rank = dist.get_rank()
    device = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(1234 + rank)  # deliberately different init per rank: DDP broadcasts rank 0's
    model = nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.BatchNorm2d(16), nn.ReLU(), nn.AdaptiveAvgPool2d(4), nn.Flatten(),
                          nn.Linear(16 * 16, 10))
    model = nn.SyncBatchNorm.convert_sync_batchnorm(model).to(device).to(memory_format=torch.channels_last)
    ddp = nn.parallel.DistributedDataParallel(model, device_ids=[device.index])
    ddp.register_comm_hook(None, default_hooks.bf16_compress_hook)
    opt = torch.optim.SGD(ddp.parameters(), lr=0.05, momentum=0.9)
    gen = torch.Generator(device=device).manual_seed(99 + rank)
    for _ in range(a.steps):
        x = torch.randn(32, 3, 16, 16, device=device, generator=gen).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (32,), device=device, generator=gen)
        loss = nn.functional.cross_entropy(ddp(x), y)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    torch.cuda.synchronize(device)
    params = [p.detach().cpu() for p in model.parameters()]
    out = os.environ.get("TRAIN_STOCK_DDP_OUT")
    if out:
        torch.save(params, os.path.join(out, f"params{rank}.pt"))
    flat = torch.cat([p.reshape(-1) for p in params]).numpy().tobytes()
    print(f"rank {rank}/{dist.get_world_size()} backend {dist.get_backend()} device {device} loss {loss.item():.4f} "
          f"params sha256 {hashlib.sha256(flat).hexdigest()[:16]}", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
