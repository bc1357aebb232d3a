"""One rank of the process-subgroup checks (spawned by tests/test_subgroups_gpu.py).

Under init_pg("b200") the rank builds the groups of ``--case`` with torchx_b200.distributed.new_group (or
new_subgroups_by_enumeration), runs the helpers on every group it belongs to, interleaved with world collectives, and
saves the results, the op counters, and the parameters of a mini-DDP + ZeRO-1 run and a SyncBatchNorm run.  ``--case
world2`` runs the same training on a plain W = 2 world, the reference for the groups of 2.  Inputs come from seeds and
the global rank; the test checks everything against the oracles."""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch import nn  # noqa: E402

N = 1031


def data(rank, seed, dtype=torch.float32, n=N):
    g = torch.Generator().manual_seed(seed * 1000 + rank)
    if dtype == torch.int64:
        return torch.randint(-(1 << 40), 1 << 40, (n,), generator=g, dtype=dtype)
    return (torch.randn(n, generator=g) * 3).to(dtype)


def bits(t):
    t = t.detach().contiguous().cpu()
    if t.dtype == torch.float32:
        return t.view(torch.int32).numpy().view(np.uint32)
    return t.numpy()


CASES = {
    "pairs": [[0, 1], [2, 3]],
    "strided": [[0, 2], [1, 3]],
    "three": [[1, 2, 3]],
    "single": [[2]],
    "twice": [[0, 1, 3], [0, 1, 3]],
    "split2x4": [[0, 1, 2, 3], [4, 5, 6, 7]],
    "split4x2": [[0, 1], [2, 3], [4, 5], [6, 7]],
}


def run_group(D, g, tag, out, rank, seed):
    """Every helper on group ``g``; world collectives in between."""
    dev = torch.device("cuda", g.comm.device)
    G, gr = g.size(), g.rank()
    x = data(rank, seed).to(dev)
    D.all_reduce(x, group=g)
    out[f"{tag}.allreduce"] = bits(x)
    y = data(rank, seed + 1, torch.int64).to(dev)
    D.all_reduce(y, op=torch.distributed.ReduceOp.MAX, group=g)
    out[f"{tag}.allreduce_max"] = bits(y)
    w = torch.full((5,), float(rank), device=dev)
    D.all_reduce(w)  # a world collective between group collectives
    out[f"{tag}.world_between"] = bits(w)
    ag = torch.empty(G * 7, dtype=torch.int32, device=dev)
    D.all_gather_into_tensor(ag, torch.arange(7, dtype=torch.int32, device=dev) + 100 * rank, group=g)
    out[f"{tag}.allgather"] = bits(ag)
    rs_in = data(rank, seed + 2, n=G * 64).to(dev)
    rs = torch.empty(64, device=dev)
    D.reduce_scatter_tensor(rs, rs_in, group=g)
    out[f"{tag}.reduce_scatter"] = bits(rs)
    b = torch.full((9,), float(rank), device=dev)
    D.broadcast(b, src=g.ranks[-1], group=g)  # a global rank
    out[f"{tag}.broadcast"] = bits(b)
    b2 = torch.full((9,), float(rank), device=dev)
    D.broadcast(b2, group=g, group_src=0)
    out[f"{tag}.broadcast_group_src"] = bits(b2)
    red = data(rank, seed + 3).to(dev)
    D.reduce(red, dst=g.ranks[0], group=g)
    if gr == 0:
        out[f"{tag}.reduce"] = bits(red)
    a2a_in = torch.arange(G * 3, dtype=torch.int32, device=dev) + 1000 * rank
    a2a = torch.empty(G * 3, dtype=torch.int32, device=dev)
    D.all_to_all_single(a2a, a2a_in, group=g)
    out[f"{tag}.alltoall"] = bits(a2a)
    if G > 1:  # a ring by global rank: send to the next member, receive from the previous one
        nxt, prv = g.ranks[(gr + 1) % G], g.ranks[(gr - 1) % G]
        msg = torch.full((11,), float(rank), device=dev)
        got = torch.empty(11, device=dev)
        ops = [D.P2POp(D.isend, msg, nxt, group=g), D.P2POp(D.irecv, got, prv, group=g)]
        for wk in D.batch_isend_irecv(ops):
            wk.wait()
        out[f"{tag}.ring"] = bits(got)
        got2 = torch.empty(11, device=dev)
        D.send(msg, nxt, group=g)  # 44 bytes: below the eager size, so every send completes before its receive
        src = D.recv(got2, group=g, group_src=(gr - 1) % G)
        out[f"{tag}.sendrecv"] = bits(got2)
        out[f"{tag}.sendrecv_src"] = np.array([src])
    gl = [torch.empty(4, device=dev) for _ in range(G)] if gr == 0 else None
    D.gather(torch.full((4,), float(rank), device=dev), gl, dst=g.ranks[0], group=g)
    if gr == 0:
        out[f"{tag}.gather"] = bits(torch.cat(gl))
    sc = torch.empty(4, device=dev)
    D.scatter(sc, [torch.full((4,), float(10 * r), device=dev) for r in range(G)] if gr == 0 else None, src=g.ranks[0], group=g)
    out[f"{tag}.scatter"] = bits(sc)
    objs = [None] * G
    D.all_gather_object(objs, {"rank": rank}, group=g)
    out[f"{tag}.objects"] = np.array([o["rank"] for o in objs])
    D.barrier(group=g)
    torch.cuda.synchronize()


def mlp(seed, dev):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(32, 64), nn.ReLU(), nn.Linear(64, 17)).to(dev)


def train(D, comm, g_rank, out, tag, group=None, world_comm=None):
    """Mini-DDP + ZeRO-1 (overlap off and on) and SyncBatchNorm on ``comm``; with ``world_comm`` a world all_reduce runs
    from a gradient hook while the group's buckets are in flight."""
    from torchx_b200.ddp import DistributedDataParallel
    from torchx_b200.ddp.zero import ZeroRedundancyOptimizer
    from torchx_b200.nn import SyncBatchNorm

    dev = torch.device("cuda", comm.device)
    for overlap in (False, True):
        model = DistributedDataParallel(mlp(5, dev), comm=comm, bucket_cap_mb=0.01, first_bucket_mb=0.005)
        opt = ZeroRedundancyOptimizer(model, torch.optim.AdamW, overlap_with_ddp=overlap, lr=1e-2)
        hooked = []
        if world_comm is not None:
            probe = torch.full((1000,), float(D.rank()), device=dev)

            def hook(p):
                D.all_reduce(probe)  # world collective issued mid-backward
                hooked.append(1)
            model.module[0].weight.register_post_accumulate_grad_hook(hook)
        for step in range(3):
            g = torch.Generator().manual_seed(100 * step + g_rank)
            x = torch.randn(8, 32, generator=g).to(dev)
            model(x).square().mean().backward()
            opt.step()
            opt.zero_grad()
        torch.cuda.synchronize()
        out[f"{tag}.params.{int(overlap)}"] = bits(torch.cat([p.detach().reshape(-1) for p in model.module.parameters()]))
        if world_comm is not None:
            out[f"{tag}.probe.{int(overlap)}"] = bits(probe)
            out[f"{tag}.hooked.{int(overlap)}"] = np.array([len(hooked)])
    torch.manual_seed(9)
    bn = SyncBatchNorm(6).to(dev)
    bn.process_group = group
    g = torch.Generator().manual_seed(500 + g_rank)
    x = (torch.randn(4, 6, 5, 5, generator=g) * 2 + 1).to(dev).requires_grad_()
    y = bn(x)
    (y * torch.arange(6, device=dev).view(1, 6, 1, 1)).sum().backward()
    torch.cuda.synchronize()
    out[f"{tag}.bn.y"] = bits(y)
    out[f"{tag}.bn.dx"] = bits(x.grad)
    out[f"{tag}.bn.running"] = bits(torch.cat([bn.running_mean, bn.running_var]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--device", type=int, required=True)
    ap.add_argument("--shm", required=True)
    ap.add_argument("--case", required=True)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    os.environ.update(RANK=str(a.rank), WORLD_SIZE=str(a.world), LOCAL_RANK=str(a.rank), B2_DEVICE=str(a.device),
                      B2_SHM_NAME=a.shm, B2_EPOCH="0")
    torch.cuda.set_device(a.device)
    import torchx_b200.distributed as D

    D.init_pg("b200", stage_mb=16)
    world = D.communicator()
    out = {}
    if a.case == "world2":
        train(D, world, a.rank, out, "train")
        np.savez(a.out, **out)
        return
    if a.case == "train":  # groups {0,1} and {2,3}, each the W = 2 world of case world2, with a world collective mid-backward
        cur, _ = D.new_subgroups(2)
        train(D, cur.comm, cur.rank(), out, "train", group=cur, world_comm=world)
        out["world.op_count"] = np.array([world.op_count])
        np.savez(a.out, **out)
        return
    if a.case in ("split2x4", "split4x2"):
        cur, groups = D.new_subgroups_by_enumeration(CASES[a.case])
        mine = [(i, g) for i, g in enumerate(groups) if isinstance(g, D.B200Group)]
        assert sum(g is not D.NON_GROUP_MEMBER for g in groups) == 1 and mine[0][1] is cur
    else:
        made = [D.new_group(r) for r in CASES[a.case]]
        mine = [(i, g) for i, g in enumerate(made) if isinstance(g, D.B200Group)]
        for g, r in zip(made, CASES[a.case]):
            assert (g is D.NON_GROUP_MEMBER) == (a.rank not in r)
    w0 = world.op_count
    world_ops = 0
    for i, g in mine:
        before = g.comm.op_count
        run_group(D, g, f"g{i}", out, a.rank, seed=7 + i)
        world_ops += 1
        out[f"g{i}.op_count"] = np.array([before, g.comm.op_count])
    # a non-member's call returns at once
    for i, g in enumerate(CASES[a.case]):
        if a.rank not in g:
            import warnings

            with warnings.catch_warnings(record=True) as ws:
                warnings.simplefilter("always")
                t = torch.zeros(3, device=f"cuda:{a.device}")
                assert D.all_reduce(t, group=D.NON_GROUP_MEMBER) is None
            assert any("does not belong to the given group" in str(w_.message) for w_ in ws)
            break
    # every rank runs the same number of world all_reduces: pad to the largest count
    most = max(sum(a_rank in g for g in CASES[a.case]) for a_rank in range(a.world))
    for _ in range(most - world_ops):
        D.all_reduce(torch.full((5,), float(a.rank), device=f"cuda:{a.device}"))
    torch.cuda.synchronize()
    out["world.op_count"] = np.array([w0, world.op_count])
    for _, g in mine:
        g.comm.close()
    D.barrier()
    np.savez(a.out, **out)


if __name__ == "__main__":
    main()
