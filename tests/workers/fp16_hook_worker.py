"""One rank of the fp16 DDP checks (spawned by tests/test_fp16_gpu.py): b200_fp16_compress_hook on STOCK
torch.nn.parallel.DistributedDataParallel, the mini-DDP with wire="f16" and with a .half() model (zero-copy bucket fill),
the mini-DDP under fp16 autocast + GradScaler with one rank forced to overflow, and - when the ranks have a GPU each - the
reference's own fp16_compress_hook over NCCL.  torch.distributed only does DDP's bookkeeping (gloo when ranks share a GPU)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
from torch import nn  # noqa: E402


def mlp(seed, half=False):
    torch.manual_seed(seed)
    # 37- and 13-wide layers: parameters that start at bucket offsets that are not vec-aligned (straddling vecs)
    m = nn.Sequential(nn.Linear(64, 256), nn.ReLU(), nn.Linear(256, 37), nn.ReLU(), nn.Linear(37, 13)).cuda()
    return m.half() if half else m


def flat_grads(m):
    g = torch.cat([p.grad.reshape(-1) for p in m.parameters()])
    return g.view(torch.int16).cpu().numpy().view(np.uint16) if g.dtype == torch.float16 else g.cpu().numpy()


def flat_params(m):
    return torch.cat([p.detach().reshape(-1).float() for p in m.parameters()]).cpu().numpy()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--device", type=int, required=True)
    ap.add_argument("--shm", required=True)
    ap.add_argument("--port", type=int, required=True)
    ap.add_argument("--backend", required=True)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()

    from torch.distributed.algorithms.ddp_comm_hooks import default_hooks
    from torch.nn.parallel import DistributedDataParallel as TorchDDP

    from torchx_b200.ddp import B200HookState, Communicator, DistributedDataParallel, b200_fp16_compress_hook

    torch.cuda.set_device(a.device)
    dist.init_process_group(a.backend, init_method=f"tcp://127.0.0.1:{a.port}", rank=a.rank, world_size=a.world)
    comm = Communicator.create(a.rank, a.world, a.device, a.shm, stage_mb=8, timeout_s=60)
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    res = {}
    x = torch.randn(32, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(100 + a.rank))

    for tag, half in (("local", False), ("local_half", True)):
        twin = mlp(0, half)
        twin(x.half() if half else x).float().square().mean().backward()
        res[tag] = flat_grads(twin)

    for tag, half in (("hook", False), ("hook_half", True)):
        m = mlp(0, half)
        d = TorchDDP(m, device_ids=[a.device], bucket_cap_mb=0.05)  # several buckets
        d.register_comm_hook(B200HookState(comm), b200_fp16_compress_hook)
        for _ in range(2):  # the second iteration runs on the rebuilt bucket layout
            d.zero_grad(set_to_none=True)
            d(x.half() if half else x).float().square().mean().backward()
        torch.cuda.synchronize()
        comm.check()
        res[tag] = flat_grads(m)

    for tag, half, wire in (("mini_f16_wire", False, "f16"), ("mini_half", True, "bf16")):  # an fp16 bucket ignores `wire`
        m = mlp(0, half)
        d = DistributedDataParallel(m, comm, bucket_cap_mb=0.05, first_bucket_mb=0.01, wire=wire)
        for _ in range(2):
            d.zero_grad(set_to_none=True)
            d(x.half() if half else x).float().square().mean().backward()
        torch.cuda.synchronize()
        comm.check()
        res[tag] = flat_grads(m)
        res[tag + "_counts"] = np.array([d.gathered_buckets, d.copied_in_buckets])

    # fp16 autocast + GradScaler + wire="f16": at step 1 rank 0 alone blows its loss up; its scaled gradients overflow the
    # fp16 wire, the sum is inf on EVERY rank, so every rank's scaler finds it, skips the step and halves the scale
    m = mlp(0)
    d = DistributedDataParallel(m, comm, bucket_cap_mb=0.05, first_bucket_mb=0.01, wire="f16")
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
    found, scales, params = [], [], []
    for step in range(4):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            loss = d(x).float().square().mean()
        if step == 1 and a.rank == 0:
            loss = loss * 1e6
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        found.append(int(sum(v.item() for v in scaler._found_inf_per_device(opt).values()) > 0))
        scaler.step(opt)
        scaler.update()
        scales.append(scaler.get_scale())
        params.append(flat_params(m))
    torch.cuda.synchronize()
    comm.check()
    res["scaler_found_inf"] = np.array(found)
    res["scaler_scale"] = np.array(scales)
    res["scaler_params"] = np.stack(params)

    if a.backend == "nccl":  # the reference's own hook over NCCL
        m3 = mlp(0)
        d3 = TorchDDP(m3, device_ids=[a.device], bucket_cap_mb=0.05)
        d3.register_comm_hook(None, default_hooks.fp16_compress_hook)
        for _ in range(2):
            d3.zero_grad(set_to_none=True)
            d3(x).square().mean().backward()
        torch.cuda.synchronize()
        res["nccl_hook"] = flat_grads(m3)
        eq = []
        for n in (1000, 65536, (1 << 20) + 3):
            buf = torch.randn(n, device="cuda", generator=torch.Generator("cuda").manual_seed(1234 + a.rank))
            ours = buf.clone()
            comm.allreduce_(ours, wire="f16")
            c = buf.to(torch.float16).div_(a.world)
            dist.all_reduce(c)
            ref = buf.clone().copy_(c)
            torch.cuda.synchronize()
            eq.append(bool(torch.equal(ours, ref)))
        res["nccl_bit_equal"] = np.array(eq)
    comm.check()
    np.savez(a.out, **res)
    dist.barrier()
    comm.close()
    dist.destroy_process_group()
    print(f"rank {a.rank} ok", flush=True)


if __name__ == "__main__":
    main()
