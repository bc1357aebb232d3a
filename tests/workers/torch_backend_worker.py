"""One rank of the "b200" torch.distributed backend checks (spawned by tests/test_torch_backend_gpu.py).

The rank first runs this package's SyncBatchNorm on the fabric under init_pg("b200"), then calls
dist.init_process_group("b200") from the environment (no gloo, no NCCL), which must share that communicator, and runs
every dist.* call (blocking, then async with waits out of issue order), stock DistributedDataParallel with and without
comm hooks, torch.nn.SyncBatchNorm, torch's ZeroRedundancyOptimizer, the mini-DDP next to group collectives, and CUDA-graph
capture.  Inputs come from seeds; outputs are saved for the test to check against the oracles."""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch import nn  # noqa: E402

FLOATS = ("float32", "bfloat16", "float16")
OPS = {"int32": ("sum", "min", "max"), "int64": ("sum", "min", "max"),
       "float32": ("sum", "avg", "min", "max"), "bfloat16": ("sum", "avg", "min", "max"), "float16": ("sum", "avg", "min", "max")}
N_REDUCE = 1031


def reduce_input(dtype, rank, seed):
    """Rank ``rank``'s input of a reduction: the test regenerates every rank's from the same formula."""
    g = torch.Generator().manual_seed(seed * 1000 + rank)
    if dtype in ("int32", "int64"):
        return torch.randint(-(1 << 30), 1 << 30, (N_REDUCE,), generator=g, dtype=getattr(torch, dtype))
    return (torch.randn(N_REDUCE, generator=g) * 3).to(getattr(torch, dtype))


def bits(t):
    t = t.detach().contiguous().cpu()
    if t.dtype in (torch.bfloat16, torch.float16):
        return t.view(torch.int16).numpy().view(np.uint16)
    if t.dtype == torch.float32:
        return t.view(torch.int32).numpy().view(np.uint32)
    return t.numpy()


def mlp(seed, dev):
    torch.manual_seed(seed)
    m = nn.Sequential(nn.Linear(64, 256), nn.ReLU(), nn.Linear(256, 37), nn.ReLU(), nn.Linear(37, 13)).to(dev)
    m.register_buffer("marker", torch.zeros(3, device=dev))
    return m


def convnet(seed, dev):
    torch.manual_seed(seed)
    net = nn.Sequential(nn.Conv2d(3, 5, 3, bias=True), nn.ReLU(), nn.Conv2d(5, 7, 3), nn.ReLU(), nn.Flatten(), nn.Linear(7 * 4 * 4, 11))
    return net.to(dev).to(memory_format=torch.channels_last)


def flat_grads(m):
    return torch.cat([p.grad.reshape(-1) for p in m.parameters()]).cpu().numpy()


def flat_params(m):
    return torch.cat([p.detach().reshape(-1).float() for p in m.parameters()]).cpu().numpy()


def collectives(dist, rank, W, dev, res, tag, async_op):
    """Every dist.* collective once; with async_op the works are waited in reverse issue order at the end."""
    works = []

    def go(w):
        if async_op:
            assert w is not None
            works.append(w)
        else:
            assert w is None
        return w

    for k, (dtype, ops) in enumerate(OPS.items()):
        for j, op in enumerate(ops):
            t = reduce_input(dtype, rank, 10 * k + j).to(dev)
            w = go(dist.all_reduce(t, op=getattr(dist.ReduceOp, op.upper()), async_op=async_op))
            if async_op and k == 0 and j == 0:
                w.wait()
                assert w.get_future().value()[0].data_ptr() == t.data_ptr()
            res[f"{tag}.allreduce.{dtype}.{op}"] = t
    x = torch.arange(7, dtype=torch.int32, device=dev) + 100 * rank
    out = torch.empty(W * 7, dtype=torch.int32, device=dev)
    go(dist.all_gather_into_tensor(out, x, async_op=async_op))
    res[f"{tag}.all_gather_into_tensor"] = out
    lst = [torch.empty(7, dtype=torch.int32, device=dev) for _ in range(W)]
    go(dist.all_gather(lst, x, async_op=async_op))
    res[f"{tag}.all_gather"] = lst
    rs_in = reduce_input("float32", rank, 77).to(dev)[: W * 100]
    rs_out = torch.empty(100, device=dev)
    go(dist.reduce_scatter_tensor(rs_out, rs_in, async_op=async_op))
    res[f"{tag}.reduce_scatter_tensor"] = rs_out
    rl_in = [reduce_input("int64", rank, 78).to(dev)[r * 50:(r + 1) * 50].clone() for r in range(W)]
    rl_out = torch.empty(50, dtype=torch.int64, device=dev)
    go(dist.reduce_scatter(rl_out, rl_in, op=dist.ReduceOp.MAX, async_op=async_op))
    res[f"{tag}.reduce_scatter"] = rl_out
    for root in range(W):
        b = torch.full((33,), float(rank * 10 + root), device=dev)
        go(dist.broadcast(b, root, async_op=async_op))
        res[f"{tag}.broadcast.{root}"] = b
        r_t = reduce_input("int64", rank, 90 + root).to(dev)
        go(dist.reduce(r_t, root, async_op=async_op))
        res[f"{tag}.reduce.{root}"] = r_t
    # all_to_all_single with uneven and zero splits: rank i sends rank j rows(i, j) rows of 3 int32s
    rows = [[(i + 2 * j) % 3 for j in range(W)] for i in range(W)]
    send = torch.cat([torch.full((rows[rank][j], 3), 1000 * rank + j, dtype=torch.int32) for j in range(W)]).to(dev)
    recv = torch.full((sum(rows[i][rank] for i in range(W)), 3), -1, dtype=torch.int32, device=dev)
    go(dist.all_to_all_single(recv, send, output_split_sizes=[rows[i][rank] for i in range(W)],
                              input_split_sizes=rows[rank], async_op=async_op))
    if async_op:
        # the input is dropped right after the call and a tensor of its size is written on the current stream at once: the
        # allocator hands it the input's block unless record_stream holds that block until the exchange has read it
        shape = send.shape
        del send
        res[f"{tag}.reuse_after_async"] = torch.full(shape, -7, dtype=torch.int32, device=dev)
    res[f"{tag}.all_to_all_single"] = recv
    outs = [torch.empty(r + 1, dtype=torch.float32, device=dev) for r in range(W)]
    ins = [torch.full((rank + 1,), float(100 * rank + j), device=dev) for j in range(W)]
    go(dist.all_to_all(outs, ins, async_op=async_op))
    res[f"{tag}.all_to_all"] = outs
    for root in (0, W - 1):
        gl = [torch.empty(5, device=dev) for _ in range(W)] if rank == root else None
        go(dist.gather(torch.full((5,), float(rank), device=dev), gl, dst=root, async_op=async_op))
        if rank == root:
            res[f"{tag}.gather.{root}"] = gl
        so = torch.empty(5, device=dev)
        sl = [torch.full((5,), float(10 * root + r), device=dev) for r in range(W)] if rank == root else None
        go(dist.scatter(so, sl, src=root, async_op=async_op))
        res[f"{tag}.scatter.{root}"] = so
    if W > 1:
        big = 4 * dist.group.WORLD.comm.p2p_eager_bytes // 4 + 17  # int32 elements: four times past the eager size
        nxt, prv = (rank + 1) % W, (rank - 1) % W
        s_t = torch.arange(big, dtype=torch.int32, device=dev) + rank
        r_t = torch.empty(big, dtype=torch.int32, device=dev)
        # the ring of torch's docs, the same op order on every rank: a send past the eager size waits for its receive, so
        # this only makes progress because the group launches the whole list as one batch
        reqs = dist.batch_isend_irecv([dist.P2POp(dist.isend, s_t, nxt), dist.P2POp(dist.irecv, r_t, prv)])
        if not async_op:
            for q in reqs:
                q.wait()
        else:
            works.extend(reqs)
        res[f"{tag}.ring"] = r_t
        small = torch.full((9,), float(rank), device=dev)
        got = torch.empty(9, device=dev)
        if async_op:
            works.append(dist.isend(small, nxt))
            works.append(dist.irecv(got, prv))
        else:
            if rank == 0:
                dist.send(small, nxt)
                dist.recv(got, prv)
            else:
                dist.recv(got, prv)
                dist.send(small, nxt)
        res[f"{tag}.sendrecv"] = got
    dist.barrier(async_op=async_op)
    for w in reversed(works):
        w.wait()


def save_collectives(res, out):
    for k, v in res.items():
        if isinstance(v, list):
            out[k] = np.stack([bits(t) for t in v]) if all(t.numel() == v[0].numel() for t in v) else \
                np.concatenate([bits(t).reshape(-1) for t in v])
        else:
            out[k] = bits(v)


def run_syncbn(m_factory, dev, rank, world, out, tag):
    import syncbn_worker as S

    for k, (name, dtype, cl, shape, sizes) in enumerate(S.CASES):
        sizes = (sizes * 2)[:world]
        if dtype == torch.bfloat16 and 0 in sizes:
            # torch's SyncBatchNorm backward: an empty rank contributes zeros of the input's dtype (bf16) to an allreduce
            # in which the other ranks' sums are fp32, so the ranks' collectives disagree under any backend
            continue
        xs, gos, w, b, rm, rv = S.case_data(k, dtype, cl, shape, sizes, dev)
        m = m_factory(shape[0]).to(dev)
        with torch.no_grad():
            m.weight.copy_(w)
            m.bias.copy_(b)
            m.running_mean.copy_(rm)
            m.running_var.copy_(rv)
        x = xs[rank].clone().requires_grad_()
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype == torch.bfloat16):
            y = m(x)
        y.backward(gos[rank])
        grad = x.grad if x.grad is not None else torch.zeros_like(x)
        for t, v in (("out", y), ("grad", grad), ("rm", m.running_mean), ("rv", m.running_var)):
            out[f"{tag}.{name}.{t}"] = bits(v)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--device", type=int, required=True)
    ap.add_argument("--shm", required=True)
    ap.add_argument("--port", type=int, required=True)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    os.environ.update(RANK=str(a.rank), WORLD_SIZE=str(a.world), LOCAL_RANK=str(a.rank), B2_DEVICE=str(a.device),
                      B2_SHM_NAME=a.shm, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(a.port))

    import torch.distributed as dist
    from torch.distributed.algorithms.ddp_comm_hooks import default_hooks
    from torch.distributed.optim import ZeroRedundancyOptimizer as TorchZero
    from torch.nn.parallel import DistributedDataParallel as TorchDDP

    import torchx_b200.distributed as D
    from torchx_b200.ddp import B200HookState, DistributedDataParallel, b200_bf16_compress_hook
    from torchx_b200.nn import SyncBatchNorm as FabricSyncBN

    rank, W = a.rank, a.world
    dev = D.init_pg("b200", stage_mb=8, timeout_s=60)
    comm = D.communicator()
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    out = {}

    # this package's SyncBatchNorm on the fabric, no process group: what torch's must match under the group
    run_syncbn(lambda c: FabricSyncBN(c, eps=1e-5, momentum=0.1), dev, rank, W, out, "sbn_fabric")
    torch.cuda.synchronize()

    dist.init_process_group("b200")
    assert dist.get_backend() == "b200" and D._COMM is comm and dist.group.WORLD.comm is comm
    assert D.local_device() == dev and dist.get_rank() == rank and dist.get_world_size() == W
    pg_stream = comm.ordered_stream
    assert pg_stream is not None

    # 1. every dist.* call, blocking then async
    for tag, async_op in (("sync", False), ("async", True)):
        res = {}
        collectives(dist, rank, W, dev, res, tag, async_op)
        torch.cuda.synchronize()
        save_collectives(res, out)
    comm.check()
    # torch's object collectives over the group
    objs = [None] * W
    dist.all_gather_object(objs, {"rank": rank, "pad": "x" * (rank * 37)})
    out["obj.all_gather"] = np.array([o["rank"] * 1000 + len(o["pad"]) for o in objs])
    bl = [f"from {rank}", rank * 3] if rank == W - 1 else [None, None]
    dist.broadcast_object_list(bl, src=W - 1)
    out["obj.broadcast"] = np.array([bl[0] == f"from {W - 1}", bl[1] == (W - 1) * 3])
    gl = [None] * W if rank == 0 else None
    dist.gather_object(("g", rank), gl, dst=0)
    if rank == 0:
        out["obj.gather"] = np.array([g[1] for g in gl])
    so = [None]
    dist.scatter_object_list(so, [("s", r * r) for r in range(W)] if rank == 0 else None, src=0)
    out["obj.scatter"] = np.array([so[0][1]])
    # helpers under the group delegate to it, async works included
    h = torch.full((5,), rank, dtype=torch.int64, device=dev)
    w = D.all_reduce(h, op=dist.ReduceOp.MAX, async_op=True)
    w.wait()
    out["helper.allreduce"] = bits(h)

    # 2. stock DDP: no hook, torch's bf16_compress_hook, b200_bf16_compress_hook on a B200HookState sharing the communicator
    x = torch.randn(32, 64, device=dev, generator=torch.Generator(dev).manual_seed(100 + rank))
    xc = torch.randn(4, 3, 8, 8, device=dev, generator=torch.Generator(dev).manual_seed(200 + rank)).contiguous(
        memory_format=torch.channels_last)
    for name, make, inp in (("mlp", mlp, x), ("conv", convnet, xc)):
        twin = make(0, dev)
        twin(inp).square().mean().backward()
        out[f"ddp.{name}.local"] = flat_grads(twin)
        for hook in ("none", "torch_bf16", "b200_bf16"):
            m = make(0, dev)
            if name == "mlp":
                m.marker.fill_(rank)
            d = TorchDDP(m, device_ids=[a.device], bucket_cap_mb=0.05 if name == "mlp" else 0.002)
            if name == "mlp":
                out[f"ddp.{name}.{hook}.marker_after_init"] = bits(m.marker)
            if hook == "torch_bf16":
                d.register_comm_hook(None, default_hooks.bf16_compress_hook)
            elif hook == "b200_bf16":
                d.register_comm_hook(B200HookState(), b200_bf16_compress_hook)
            opt = torch.optim.SGD(d.parameters(), lr=0.1)
            for _ in range(2):  # the second iteration runs on the rebuilt buckets
                if name == "mlp":
                    m.marker.fill_(rank)
                d.zero_grad(set_to_none=True)
                d(inp).square().mean().backward()
            torch.cuda.synchronize()
            out[f"ddp.{name}.{hook}.grads"] = flat_grads(m)
            if name == "mlp":
                out[f"ddp.{name}.{hook}.marker"] = bits(m.marker)
            opt.step()
            torch.cuda.synchronize()
            out[f"ddp.{name}.{hook}.params"] = flat_params(m)
    comm.check()

    # 3. torch.nn.SyncBatchNorm under the group
    run_syncbn(lambda c: nn.SyncBatchNorm(c, eps=1e-5, momentum=0.1), dev, rank, W, out, "sbn_torch")

    # 4. torch's ZeroRedundancyOptimizer over stock DDP, against the unsharded optimizer over stock DDP
    xz = torch.randn(16, 64, device=dev, generator=torch.Generator(dev).manual_seed(300 + rank))
    for name, zero in (("plain", False), ("zero", True)):
        m = mlp(1, dev)
        d = TorchDDP(m, device_ids=[a.device])
        if zero:
            opt = TorchZero(d.parameters(), optimizer_class=torch.optim.AdamW, lr=1e-2, weight_decay=0.01)
        else:
            opt = torch.optim.AdamW(d.parameters(), lr=1e-2, weight_decay=0.01)
        for _ in range(3):
            opt.zero_grad(set_to_none=True)
            d(xz).square().mean().backward()
            opt.step()
        torch.cuda.synchronize()
        out[f"zero.{name}"] = flat_params(m)
        if zero:
            opt.consolidate_state_dict(to=0)
            if rank == 0:
                sd = opt.state_dict()
                out["zero.consolidated_steps"] = np.array([float(s["step"]) for s in sd["state"].values()])
    comm.check()

    # 5. the mini-DDP after init_process_group: it takes over the ordered stream; dist.* calls before, between and after
    #    its backwards, torch's SyncBatchNorm inside the wrapped model; one communicator throughout
    def sbn_model():
        torch.manual_seed(5)
        return nn.Sequential(nn.Linear(24, 40), nn.SyncBatchNorm(40), nn.ReLU(), nn.Linear(40, 9)).to(dev)

    xm = torch.randn(8 + rank, 24, device=dev, generator=torch.Generator(dev).manual_seed(400 + rank))
    pending = torch.full((1000,), float(rank), device=dev)
    w_pending = dist.all_reduce(pending, async_op=True)  # still queued on the group's stream when the mini-DDP takes over
    ref = sbn_model()
    dref = DistributedDataParallel(ref, wire="f32", bucket_cap_mb=0.002, first_bucket_mb=0.001)
    assert dref.comm is comm and comm.ordered_stream is not pg_stream
    w_pending.wait()
    out["mini.pending"] = bits(pending)
    with dref.no_sync():
        dref(xm).square().mean().backward()
    torch.cuda.synchronize()
    out["mini.local"] = flat_grads(ref)
    m = sbn_model()
    dm = DistributedDataParallel(m, wire="f32", bucket_cap_mb=0.002, first_bucket_mb=0.001)
    counts = []
    for step in range(2):
        a1 = torch.full((3,), float(rank + step), device=dev)
        dist.all_reduce(a1)
        dm.zero_grad(set_to_none=True)
        loss = dm(xm).square().mean()
        before = comm.op_count
        loss.backward()
        a2 = torch.full((3,), float(rank), dtype=torch.float32, device=dev)
        dist.all_reduce(a2, op=dist.ReduceOp.MAX)
        torch.cuda.synchronize()
        counts.append(comm.op_count - before)
        out[f"mini.a1.{step}"] = bits(a1)
        out[f"mini.a2.{step}"] = bits(a2)
    out["mini.grads"] = flat_grads(m)
    out["mini.op_counts"] = np.array(counts)
    out["mini.buckets"] = np.array(len(dm.buckets))
    comm.check()
    # an async group collective still pending while a mini-DDP forward broadcasts its buffers: the broadcast runs after it
    bn_m = nn.Sequential(nn.Linear(24, 16), nn.BatchNorm1d(16)).to(dev)
    dbn = DistributedDataParallel(bn_m, wire="f32")
    bn_m[1].num_batches_tracked.fill_(10 * rank + 5)  # the forward's buffer broadcast brings rank 0's back
    pend = torch.full((1 << 22,), float(rank + 1), device=dev)
    w = dist.all_reduce(pend, async_op=True)
    dbn(xm)
    w.wait()
    torch.cuda.synchronize()
    out["mini.async_forward.allreduce"] = bits(pend[:: 1 << 12])
    out["mini.async_forward.nbt"] = bits(bn_m[1].num_batches_tracked)
    comm.check()

    # 7. CUDA-graph capture: every group collective refuses before enqueuing anything
    t = torch.zeros(8, device=dev)
    before = comm.op_count
    refused = []
    s = torch.cuda.Stream(device=dev)
    for fn in (lambda: dist.all_reduce(t), lambda: dist.broadcast(t, 0), lambda: dist.barrier()):
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g, stream=s):
                fn()
        except RuntimeError as e:
            refused.append("cannot be captured" in str(e))
    torch.cuda.synchronize()
    out["capture.refused"] = np.array(refused)
    out["capture.op_delta"] = np.array(comm.op_count - before)
    dist.all_reduce(t)  # the communicator still works
    torch.cuda.synchronize()

    # 6. lifecycle: destroy and re-init in the same process, on the same communicator
    dist.destroy_process_group()
    assert D._COMM is comm and not dist.is_initialized()
    dist.init_process_group("b200")
    assert dist.group.WORLD.comm is comm
    t = torch.full((4,), float(rank + 1), device=dev)
    dist.all_reduce(t)
    torch.cuda.synchronize()
    out["reinit.allreduce"] = bits(t)
    comm.check()
    np.savez(a.out, **out)
    dist.barrier()
    dist.destroy_process_group()
    comm.close()
    print(f"rank {rank} ok", flush=True)


if __name__ == "__main__":
    main()
