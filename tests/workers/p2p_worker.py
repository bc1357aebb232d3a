"""One rank of the point-to-point checks (spawned by tests/test_p2p_gpu.py).

--backend b200: the public path of a training script under init_pg("b200"), with no torch.distributed process group
anywhere: send / recv, isend / irecv with wait(), batch_isend_irecv built from P2POp, gather and scatter.  `expected` is
what each rank must end with.
--backend nccl: one GPU per rank: NCCL's batch_isend_irecv and the native communicator on the same inputs."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def block(src, dst, n, dtype):
    """What rank src gives rank dst: values that name the pair and the position."""
    return (1000 * src + 100 * dst + np.arange(n)).astype(dtype)


def expected(rank, world):
    peer = 1 - rank
    return {
        "recv": block(peer, rank, 37, np.int64),
        "irecv": block(peer, rank, 3 << 18, np.float32),  # above one chunk
        "batch_a": block(peer, rank, 5, np.float64),
        "batch_b": block(peer, rank, 1 << 21, np.int32),  # above the eager size: needs the batch to make progress
        "gather": np.stack([block(q, 0, 6, np.int32) for q in range(world)]) if rank == 0 else np.zeros(0, np.int32),
        "scatter": block(1, rank, 9, np.float32),
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
    peer = 1 - rank

    def dev(x):
        return torch.from_numpy(np.ascontiguousarray(x)).to(device)

    # send / recv: rank 0 sends first, rank 1 receives first (a 296-byte message is eager)
    out = torch.empty(37, dtype=torch.int64, device=device)
    if rank == 0:
        D.send(dev(block(0, 1, 37, np.int64)), 1)
        assert D.recv(out, 1) == 1
    else:
        assert D.recv(out, 0) == 0
        D.send(dev(block(1, 0, 37, np.int64)), 0)
    res["recv"] = out.cpu().numpy()

    out = torch.empty(3 << 18, device=device)
    works = [D.isend(dev(block(rank, peer, 3 << 18, np.float32)), peer), D.irecv(out, peer)]
    assert all(w.wait() is True for w in works)
    res["irecv"] = out.cpu().numpy()
    assert all(w.is_completed() for w in works)

    a_out = torch.empty(5, dtype=torch.float64, device=device)
    b_out = torch.empty(1 << 21, dtype=torch.int32, device=device)
    # on each channel the messages match in issue order (first the float64 one, then the int32 one), but the two ranks
    # interleave their sends and receives differently
    send_a = D.P2POp(D.isend, dev(block(rank, peer, 5, np.float64)), peer)
    send_b = D.P2POp(dist.isend, dev(block(rank, peer, 1 << 21, np.int32)), peer)
    recv_a, recv_b = D.P2POp(D.irecv, a_out, peer), D.P2POp(dist.irecv, b_out, peer)
    ops = [send_a, recv_a, send_b, recv_b] if rank == 0 else [recv_a, recv_b, send_a, send_b]
    for w in D.batch_isend_irecv(ops):
        w.wait()
    res["batch_a"], res["batch_b"] = a_out.cpu().numpy(), b_out.cpu().numpy()

    t = dev(block(rank, 0, 6, np.int32))
    if rank == 0:
        lst = [torch.empty(6, dtype=torch.int32, device=device) for _ in range(world)]
        D.gather(t, lst, dst=0)
        res["gather"] = torch.stack(lst).cpu().numpy()
    else:
        D.gather(t, dst=0)
        res["gather"] = np.zeros(0, np.int32)

    out = torch.empty(9, device=device)
    D.scatter(out, [dev(block(1, q, 9, np.float32)) for q in range(world)] if rank == 1 else None, src=1)
    res["scatter"] = out.cpu().numpy()

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
    peer = 1 - a.rank
    eq = []
    g = torch.Generator().manual_seed(31 + a.rank)
    for dtype in (torch.uint8, torch.bfloat16, torch.float32, torch.float64, torch.int64):
        e = torch.empty(0, dtype=dtype).element_size()
        for n in (1, 4099, (5 << 20) + 3):  # elements: up to above the eager size
            xs = [torch.randint(0, 256, (n * e + k * e,), generator=g, dtype=torch.uint8).to(device).view(dtype) for k in range(2)]
            want = [torch.empty(n + k, dtype=dtype, device=device) for k in range(2)]
            got = [torch.empty_like(t) for t in want]
            works = dist.batch_isend_irecv([dist.P2POp(dist.isend, xs[0], peer), dist.P2POp(dist.irecv, want[0], peer),
                                            dist.P2POp(dist.isend, xs[1], peer), dist.P2POp(dist.irecv, want[1], peer)])
            for w in works:
                w.wait()
            comm.p2p_([("send", xs[0], peer), ("recv", got[0], peer), ("send", xs[1], peer), ("recv", got[1], peer)])
            torch.cuda.synchronize()
            comm.check()
            eq.append(all(torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(got, want)))
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
