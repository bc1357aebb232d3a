"""One rank of the exact-collective checks (spawned by tests/test_exact_ops_gpu.py): the public path of a training script
under init_pg("b200") - the reference's compute_world_size (an int64 one-hot summed with all_reduce), a float MAX, and
all_gather_into_tensor / all_gather - with no torch.distributed process group anywhere."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--device", type=int, required=True)
    ap.add_argument("--shm", required=True)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    os.environ.update(RANK=str(a.rank), WORLD_SIZE=str(a.world), LOCAL_RANK=str(a.rank), B2_DEVICE=str(a.device),
                      B2_SHM_NAME=a.shm)

    import torch.distributed as dist

    import torchx_b200.distributed as D

    device = D.init_pg("b200", stage_mb=8, timeout_s=60)
    comm = D.communicator()
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    assert not dist.is_initialized()
    rank, world = D.rank(), D.world_size()
    res = {}

    # the reference's compute_world_size (torchx/examples/apps/compute_world_size/module/util.py)
    t = F.one_hot(torch.tensor(rank), num_classes=world).to(device)
    assert t.dtype == torch.int64
    D.all_reduce(t)
    res["one_hot"] = t.cpu().numpy()
    res["computed_world_size"] = np.array(int(torch.sum(t).item()))

    # the slowest rank's time, an early-stopping flag, a NaN that must reach every rank
    x = torch.tensor([0.5 + rank, -float(rank), float("nan") if rank == world - 1 else 1.0, -0.0 if rank == 0 else 0.0],
                     device=device)
    D.all_reduce(x, op=dist.ReduceOp.MAX)
    res["max"] = x.cpu().numpy()

    inp = torch.arange(5, dtype=torch.int32, device=device) + 10 * rank
    out = torch.empty(world * 5, dtype=torch.int32, device=device)
    D.all_gather_into_tensor(out, inp)
    res["gather_into_tensor"] = out.cpu().numpy()
    lst = [torch.empty(5, dtype=torch.int32, device=device) for _ in range(world)]
    D.all_gather(lst, inp)
    res["gather_list"] = torch.stack(lst).cpu().numpy()

    torch.cuda.synchronize()
    comm.check()
    np.savez(a.out, **res)
    D.barrier()
    comm.close()
    print(f"rank {a.rank} ok", flush=True)


if __name__ == "__main__":
    main()
