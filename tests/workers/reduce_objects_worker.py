"""One rank of the reduce and object-collective checks (spawned by tests/test_reduce_gpu.py and
tests/test_object_collectives_gpu.py).

--backend b200: the public path of a training script under init_pg("b200"), with no torch.distributed process group:
reduce with root 1, then all six object collectives, through torchx_b200.distributed.
--backend gloo: the same script through the same functions with a 2-rank gloo process group on CPU tensors, where every
one of them is torch.distributed's own: the reference the b200 results must equal.
--backend nccl: one GPU per rank: NCCL's reduce and the native communicator's reduce_ on the same inputs.

Results are written as a pickled dict of plain values: tensors become (dtype, device type, list)."""
import argparse
import os
import pickle
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = 1
BIG = 5 << 20  # bytes: larger than the fabric's eager point-to-point limit (8 x 512 KiB)


def plain(x):
    """x with every tensor replaced by (dtype, device type, values) and every container rebuilt, for comparison."""
    if isinstance(x, torch.Tensor):
        return (str(x.dtype), x.device.type, x.detach().cpu().tolist())
    if isinstance(x, dict):
        return {k: plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(plain(v) for v in x)
    return x


def values(t):
    """A reduced tensor as (dtype, values): the b200 run reduces CUDA tensors, the gloo run CPU ones."""
    return (str(t.dtype), t.cpu().tolist())


def big_bytes(rank):
    return np.random.default_rng(100 + rank).integers(0, 256, BIG, dtype=np.uint8).tobytes()


def scenario(D, device, res, on_fabric):
    import torch.distributed as dist

    rank, world = D.rank(), D.world_size()
    cuda = torch.device("cuda", torch.cuda.current_device())

    # ---- reduce to rank 1 ----
    a = torch.tensor([rank + 1, 10 * rank - 3, (1 << 62) + rank, -(1 << 62)], dtype=torch.int64, device=device)
    D.reduce(a, ROOT)
    res["reduce_int64_sum"] = values(a)
    b = torch.tensor([5 - rank, -7 * rank, 2**31 - 1, -(2**31) + rank], dtype=torch.int32, device=device)
    D.reduce(b, dst=ROOT, op=dist.ReduceOp.MIN)
    res["reduce_int32_min"] = values(b)
    c = torch.tensor([0.1 * (rank + 1), -1.5, 3e38, 1e-3 * rank], dtype=torch.float32, device=device)
    D.reduce(c, ROOT, op=dist.ReduceOp.SUM)
    res["reduce_float32_sum"] = values(c)
    if on_fabric:  # gloo has no AVG and promises nothing for a NaN under MIN / MAX: checked against written-out values
        m = torch.tensor([float(rank), float("nan") if rank == 1 else -0.0, -0.0 if rank == 0 else 0.0, -1.0 - rank],
                         device=device)
        D.reduce(m, ROOT, op=dist.ReduceOp.MAX)
        res["reduce_float32_max_nan"] = values(m)
        v = torch.tensor([1.0, 3.0, -0.25], dtype=torch.bfloat16, device=device) * (rank + 1)
        D.reduce(v, ROOT, op=dist.ReduceOp.AVG)
        res["reduce_bf16_avg"] = values(v)

    # ---- the object collectives ----
    mine = {"rank": rank, "metrics": [1.5 * rank, None], "nested": {"t": torch.arange(3) + rank, "s": "r" * rank}}
    out = [None] * world
    D.all_gather_object(out, mine)
    res["all_gather_object"] = plain(out)

    objs = ["/runs/exp-7", 1234, {"seed": 42, "cuda": torch.full((2,), 7.0, device=cuda)}] if rank == ROOT else [None] * 3
    D.broadcast_object_list(objs, src=ROOT)
    res["broadcast_object_list"] = plain(objs)

    gl = [None] * world if rank == ROOT else None
    D.gather_object({"from": rank, "big": big_bytes(rank) if rank == 0 else b""}, gl, dst=ROOT)
    res["gather_object"] = plain(gl)

    so = [None]
    D.scatter_object_list(so, [{"to": 0, "big": big_bytes(7)}, [None, ()]] if rank == ROOT else None, src=ROOT)
    res["scatter_object_list"] = plain(so)

    if rank == 0:
        D.send_object_list([big_bytes(3), {"cuda": torch.arange(4, device=cuda)}, None], dst=1)
        back = [None]
        res["recv_object_list_src"] = D.recv_object_list(back, src=1)
        res["recv_object_list"] = plain(back)
    else:
        got = [None] * 3
        res["recv_object_list_src"] = D.recv_object_list(got, src=0)
        res["recv_object_list"] = plain(got)
        D.send_object_list([[]], dst=0)


def native(a, res):
    import torch.distributed as dist

    import torchx_b200.distributed as D

    device = D.init_pg("b200", stage_mb=8, timeout_s=60)
    torch.cuda.set_device(device)
    comm = D.communicator()
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    assert not dist.is_initialized()
    scenario(D, device, res, on_fabric=True)
    torch.cuda.synchronize()
    comm.check()
    D.barrier()
    comm.close()


def with_gloo(a, res):
    import torch.distributed as dist

    import torchx_b200.distributed as D

    torch.cuda.set_device(a.device)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{a.port}", rank=a.rank, world_size=a.world)
    scenario(D, torch.device("cpu"), res, on_fabric=False)
    dist.barrier()
    dist.destroy_process_group()


def against_nccl(a, res):
    import torch.distributed as dist

    from torchx_b200.ddp import Communicator

    torch.cuda.set_device(a.device)
    device = torch.device("cuda", a.device)
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{a.port}", rank=a.rank, world_size=a.world)
    comm = Communicator.create(a.rank, a.world, a.device, a.shm, stage_mb=8, timeout_s=60)
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    eq = {}
    ops = {"sum": dist.ReduceOp.SUM, "avg": dist.ReduceOp.AVG, "min": dist.ReduceOp.MIN, "max": dist.ReduceOp.MAX}
    for dtype in (torch.float32, torch.bfloat16, torch.float16, torch.int32, torch.int64):
        for name, op in ops.items():
            if name == "avg" and not dtype.is_floating_point:
                continue
            g = torch.Generator().manual_seed(17 + a.rank)
            n = 4099 * a.world
            if dtype.is_floating_point:
                t = torch.randn(n, generator=g).to(dtype).to(device)
            else:
                t = torch.randint(-(1 << 30), 1 << 30, (n,), generator=g, dtype=dtype).to(device)
            for root in range(a.world):
                want, got = t.clone(), t.clone()
                dist.reduce(want, root, op=op)
                comm.reduce_(got, root, name)
                torch.cuda.synchronize()
                comm.check()
                ints = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[got.element_size()]
                eq[f"{dtype} {name} root {root}"] = bool(torch.equal(got.view(ints), want.view(ints)))
    res["nccl_bit_equal"] = eq
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
    ap.add_argument("--backend", choices=("b200", "gloo", "nccl"), default="b200")
    ap.add_argument("--port", type=int, default=0)
    a = ap.parse_args()
    os.environ.update(RANK=str(a.rank), WORLD_SIZE=str(a.world), LOCAL_RANK=str(a.rank), B2_DEVICE=str(a.device),
                      B2_SHM_NAME=a.shm)
    res = {}
    {"b200": native, "gloo": with_gloo, "nccl": against_nccl}[a.backend](a, res)
    with open(a.out, "wb") as f:
        pickle.dump(res, f)
    print(f"rank {a.rank} ok", flush=True)


if __name__ == "__main__":
    main()
