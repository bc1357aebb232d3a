"""Memory of the mini-DDP with and without ZeRO-1 (``ZeroRedundancyOptimizer``), GPT-2-small with AdamW.

Two parts:

  * exact per-rank optimizer-state bytes at W = 1, 2 and 4, from the parameter shapes and the bucket plan alone (no GPU:
    ``--cpu-only``): AdamW keeps exp_avg and exp_avg_sq, 8 B per fp32 element it steps, and a sharded rank steps the
    elements of its block of every bucket that belong to a parameter (not the pad);
  * on a GPU: ``torch.cuda.max_memory_allocated`` over two training steps with W ranks sharing the one device (so the
    figure is the device's total for all W ranks), sharded and unsharded, and the W = 1 step time both ways.

    python tools/zero_memory.py --cpu-only
    python tools/zero_memory.py [--batch 2] [--seq 1024] [--steps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

WORLDS = (1, 2, 4)


def gpt2(device="cpu"):
    import transformers

    transformers.logging.set_verbosity_error()
    torch.manual_seed(0)
    with torch.device(device):
        return transformers.GPT2LMHeadModel(transformers.GPT2Config())


def state_bytes(model, world: int) -> dict:
    """Exact AdamW state bytes per rank (the most any rank holds), unsharded and sharded, with the mini-DDP's default
    bucket plan (1 MiB first bucket, 25 MiB buckets)."""
    from torchx_b200.ddp.bucketing import MIB, plan_buckets
    from torchx_b200.ddp.zero import block_intersections, padded_block

    params = [p for p in model.parameters() if p.requires_grad]
    specs = plan_buckets([p.numel() for p in params], [p.element_size() for p in params], [str(p.dtype) for p in params],
                         1 * MIB, 25 * MIB)
    n = sum(p.numel() for p in params)
    per_rank = [0] * world
    for s in specs:
        B = padded_block(s.numel, world)
        for r in range(world):
            per_rank[r] += sum(hi - lo for _, lo, hi in block_intersections(s.offsets, s.numels, B, r))
    assert sum(per_rank) == n
    return {"world": world, "params": n, "unsharded_state_bytes": 8 * n, "sharded_state_bytes": 8 * max(per_rank)}


def measure(world: int, sharded: bool, batch: int, seq: int, steps: int) -> dict:
    """Peak allocated device memory over `steps` training steps of W ranks sharing cuda:0, and the mean step time."""
    from torchx_b200.ddp import Communicator, DistributedDataParallel, ZeroRedundancyOptimizer

    torch.cuda.empty_cache()
    if world > 1:
        # The constructors broadcast rank 0's parameters in chunks, with a cat / copy between them; the ranks are issued
        # from this one thread, and the first launch of a kernel (lazy module loading) would wait behind rank 0's first
        # broadcast, which rank 1 has not joined yet.  So run the same chunking once with a broadcast that does nothing.
        import types

        stub = types.SimpleNamespace(world_size=world, comm=types.SimpleNamespace(rank=1, broadcast_=lambda t, root: t))
        m = gpt2("cuda")
        DistributedDataParallel._broadcast_coalesced(stub, [p.data for p in m.parameters()] + [b.data for b in m.buffers()])
        del m
        torch.cuda.synchronize()
    comms = Communicator.create_local([0] * world, stage_mb=64)
    for c in comms:
        c.set_timeout(60.0)
        c.set_max_ctas(max(1, 64 // world))
    streams = [torch.cuda.Stream() for _ in range(world)]
    models, opts = [], []
    try:
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                # one algorithm for every bucket: the ranks are issued from this one thread, and a kernel's first launch
                # (lazy module loading) must not wait behind a collective of rank 0 that rank 1 has not joined yet
                models.append(DistributedDataParallel(gpt2("cuda"), comms[r], broadcast_buffers=False,
                                                      algo="twoshot" if world > 1 else "auto"))
        torch.cuda.synchronize()
        for m in models:
            if sharded:
                opts.append(ZeroRedundancyOptimizer(m, torch.optim.AdamW, lr=1e-4, weight_decay=0.1))
            else:
                opts.append(torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0.1))
        g = torch.Generator().manual_seed(0)
        xs = [torch.randint(0, 50257, (batch, seq), generator=g).cuda() for _ in range(world)]

        def phase(fn):
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    fn(r)
            torch.cuda.synchronize()

        def backward(r):
            opts[r].zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = models[r](xs[r], labels=xs[r]).loss
            loss.backward()

        def local_backward(r):
            with models[r].no_sync():
                backward(r)

        phase(local_backward)  # loads every compute kernel with no collective in flight
        torch.cuda.reset_peak_memory_stats()
        times = []
        for _ in range(steps):
            t0 = time.perf_counter()
            phase(backward)
            phase(lambda r: opts[r].step())
            times.append(time.perf_counter() - t0)
        for c in comms:
            c.check()
        return {"world": world, "sharded": sharded, "batch": batch, "seq": seq,
                "max_memory_allocated_bytes": torch.cuda.max_memory_allocated(),
                "step_ms": round(1e3 * sum(times[1:]) / max(1, len(times) - 1), 2) if world == 1 else None}
    finally:
        del models, opts
        for c in comms:
            c.close()
        torch.cuda.synchronize()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpu-only", action="store_true", help="only the exact optimizer-state bytes (no GPU)")
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--seq", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    model = gpt2("meta")
    for w in WORLDS:
        print(json.dumps({"kind": "state_bytes", **state_bytes(model, w)}), flush=True)
    if args.cpu_only:
        return
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    print(json.dumps({"kind": "device", "name": torch.cuda.get_device_name(0)}), flush=True)
    for w in WORLDS:
        for sharded in (False, True):
            print(json.dumps({"kind": "memory", **measure(w, sharded, args.batch, args.seq, args.steps)}), flush=True)


if __name__ == "__main__":
    main()
