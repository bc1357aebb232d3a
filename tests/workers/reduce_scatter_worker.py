"""One rank of the reduce-scatter checks (spawned by tests/test_reduce_scatter_gpu.py).

--backend b200: the public path of a training script under init_pg("b200"), with no torch.distributed process group
anywhere: reduce_scatter_tensor, reduce_scatter (the list form) and broadcast(src=1).
--backend nccl: one GPU per rank: NCCL's reduce_scatter_tensor and the native communicator on the same inputs."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

N_PER_RANK = 4099  # not a multiple of a vec: every block but the first starts misaligned


def inputs(rank, world, dtype, device):
    g = torch.Generator().manual_seed(17 + rank)
    if dtype.is_floating_point:
        return torch.randn(world * N_PER_RANK, generator=g).to(dtype).to(device)
    return torch.randint(-(1 << 30), 1 << 30, (world * N_PER_RANK,), generator=g, dtype=dtype).to(device)


def native(a, res):
    import torch.distributed as dist

    import torchx_b200.distributed as D

    device = D.init_pg("b200", stage_mb=8, timeout_s=60)
    comm = D.communicator()
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    assert not dist.is_initialized()
    rank, world = D.rank(), D.world_size()

    # the per-rank share of a summed metric: rank r contributes r + 1 to every block
    t = torch.full((world, 3), rank + 1, dtype=torch.int64, device=device) * torch.arange(1, world + 1, device=device)[:, None]
    out = torch.empty(3, dtype=torch.int64, device=device)
    D.reduce_scatter_tensor(out, t)
    res["rs_tensor_sum"] = out.cpu().numpy()
    x = torch.tensor([[float(rank), -float(rank)], [0.5 * rank, float("nan") if rank == 1 else 1.0]], device=device)
    y = torch.empty(2, device=device)
    D.reduce_scatter_tensor(y, x, op=dist.ReduceOp.MAX)
    res["rs_tensor_max"] = y.cpu().numpy()
    z = torch.empty(2, device=device)
    D.reduce_scatter_tensor(z, x, op=dist.ReduceOp.AVG)
    res["rs_tensor_avg"] = z.cpu().numpy()

    lst = [torch.arange(4, dtype=torch.int32, device=device).view(2, 2) * (q + 1) + 100 * rank for q in range(world)]
    o = torch.empty(2, 2, dtype=torch.int32, device=device)
    D.reduce_scatter(o, lst)
    res["rs_list_sum"] = o.cpu().numpy()
    o2 = torch.empty(2, 2, dtype=torch.int32, device=device)
    D.reduce_scatter(o2, lst, op=dist.ReduceOp.MIN)
    res["rs_list_min"] = o2.cpu().numpy()

    seed = torch.tensor([1000 + rank, 7], dtype=torch.int64, device=device)
    D.broadcast(seed, src=1)
    res["broadcast"] = seed.cpu().numpy()
    w = torch.full((5,), float(rank), dtype=torch.bfloat16, device=device)
    D.broadcast(w, 1)
    res["broadcast_bf16"] = w.float().cpu().numpy()

    torch.cuda.synchronize()
    comm.check()
    D.barrier()
    comm.close()


def against_nccl(a, res):
    import torch.distributed as dist

    from torchx_b200.ddp import Communicator

    torch.cuda.set_device(a.device)
    device = torch.device("cuda", a.device)
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{a.port}", rank=a.rank, world_size=a.world)
    comm = Communicator.create(a.rank, a.world, a.device, a.shm, stage_mb=8, timeout_s=60)
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    eq = []
    ops = {"sum": dist.ReduceOp.SUM, "min": dist.ReduceOp.MIN, "max": dist.ReduceOp.MAX}
    for dtype in (torch.float32, torch.bfloat16, torch.float16, torch.int32, torch.int64):
        for name, op in ops.items():
            t = inputs(a.rank, a.world, dtype, device)
            want = torch.empty(N_PER_RANK, dtype=dtype, device=device)
            dist.reduce_scatter_tensor(want, t, op=op)
            got = torch.empty(N_PER_RANK, dtype=dtype, device=device)
            comm.reduce_scatter_(got, t, name)
            torch.cuda.synchronize()
            comm.check()
            ints = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[got.element_size()]
            eq.append(bool(torch.equal(got.view(ints), want.view(ints))))
    res["nccl_bit_equal"] = np.array(eq)
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--device", type=int, required=True)
    ap.add_argument("--shm", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--backend", choices=("b200", "nccl"), default="b200")
    ap.add_argument("--port", type=int, default=0)
    a = ap.parse_args()
    os.environ.update(RANK=str(a.rank), WORLD_SIZE=str(a.world), LOCAL_RANK=str(a.rank), B2_DEVICE=str(a.device),
                      B2_SHM_NAME=a.shm)
    res = {}
    if a.backend == "b200":
        native(a, res)
    else:
        against_nccl(a, res)
    np.savez(a.out, **res)
    print(f"rank {a.rank} ok", flush=True)


if __name__ == "__main__":
    main()
