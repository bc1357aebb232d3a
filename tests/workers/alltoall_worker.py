"""One rank of the all-to-all checks (spawned by tests/test_alltoall_gpu.py).

--backend b200: the public path of a training script under init_pg("b200"), with no torch.distributed process group
anywhere: all_to_all_single without and with split sizes, and all_to_all.  `expected` is what each rank must end with.
--backend nccl: one GPU per rank: NCCL's all_to_all_single and the native communicator on the same inputs."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def rows(j, r):
    """Rows rank j sends rank r in the split case: 0 for some pairs."""
    return (3 * j + 2 * r) % 5


def block(j, r, n, cols, dtype):
    """The n x cols block rank j sends rank r: values that name the pair and the position."""
    return (1000 * j + 100 * r + np.arange(n * cols).reshape(n, cols)).astype(dtype)


def expected(rank, world):
    return {
        "single_even": np.concatenate([block(q, rank, 3, 2, np.int64) for q in range(world)]),
        "single_split": np.concatenate([block(q, rank, rows(q, rank), 3, np.float32) for q in range(world)]),
        "single_split_idle": np.concatenate([block(q, rank, 0 if 0 in (q, rank) else 2, 5, np.float64) for q in range(world)]),
        **{f"list_{q}": block(q, rank, q + 1, rank + 1, np.int32) for q in range(world)},
    }


def native(a, res):
    import torch.distributed as dist

    import torchx_b200.distributed as D

    device = D.init_pg("b200", stage_mb=8, timeout_s=60)
    comm = D.communicator()
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    assert not dist.is_initialized()
    rank, world = D.rank(), D.world_size()

    def dev(x):
        return torch.from_numpy(np.ascontiguousarray(x)).to(device)

    inp = dev(np.concatenate([block(rank, q, 3, 2, np.int64) for q in range(world)]))
    out = torch.empty(world * 3, 2, dtype=torch.int64, device=device)
    D.all_to_all_single(out, inp)
    res["single_even"] = out.cpu().numpy()

    send = [rows(rank, q) for q in range(world)]
    recv = [rows(q, rank) for q in range(world)]
    inp = dev(np.concatenate([block(rank, q, send[q], 3, np.float32) for q in range(world)]))
    out = torch.empty(sum(recv), 3, device=device)
    D.all_to_all_single(out, inp, output_split_sizes=recv, input_split_sizes=send)
    res["single_split"] = out.cpu().numpy()

    # rank 0 sends and receives nothing while the others exchange
    send = [0 if 0 in (rank, q) else 2 for q in range(world)]
    inp = dev(np.concatenate([block(rank, q, send[q], 5, np.float64) for q in range(world)]))
    out = torch.empty(sum(send), 5, dtype=torch.float64, device=device)
    D.all_to_all_single(out, inp, send, send)
    res["single_split_idle"] = out.cpu().numpy()

    outs = [torch.empty(q + 1, rank + 1, dtype=torch.int32, device=device) for q in range(world)]
    D.all_to_all(outs, [dev(block(rank, q, rank + 1, q + 1, np.int32)) for q in range(world)])
    for q, t in enumerate(outs):
        res[f"list_{q}"] = t.cpu().numpy()

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
    comm = Communicator.create(a.rank, a.world, a.device, a.shm, stage_mb=64, timeout_s=60)
    comm.set_timeout(30.0)
    eq = []
    g = torch.Generator().manual_seed(29 + a.rank)
    for dtype in (torch.uint8, torch.bfloat16, torch.float32, torch.float64, torch.int64):
        for split in (False, True):
            rows_in = 4099 if split else 4096  # rows of 3 elements per rank
            S = [[1, rows_in - 1], [5, rows_in - 5]]  # S[j][q]: rows rank j sends rank q
            send = S[a.rank] if split else None
            recv = [S[0][a.rank], S[1][a.rank]] if split else None
            x = torch.randint(0, 256, (rows_in, 3 * torch.empty(0, dtype=dtype).element_size()), generator=g,
                              dtype=torch.uint8).to(device).view(dtype)  # random bits: NaNs with any payload included
            out_rows = sum(recv) if split else rows_in
            want = torch.empty(out_rows, 3, dtype=dtype, device=device)
            dist.all_to_all_single(want, x, output_split_sizes=recv, input_split_sizes=send)
            got = torch.empty_like(want)
            comm.alltoall_(list(torch.split(got, recv or [out_rows // 2] * 2)), list(torch.split(x, send or [rows_in // 2] * 2)))
            torch.cuda.synchronize()
            comm.check()
            eq.append(bool(torch.equal(got.view(torch.uint8), want.view(torch.uint8))))
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
