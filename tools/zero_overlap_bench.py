"""ZeRO-1 with the optimizer step inside the backward's reduce-scatter (``overlap_with_ddp=True``) against the unsharded
mini-DDP and the plain sharded one, GPT-2-small, AdamW(fused=True), bf16 autocast.

Three configurations: ``unsharded`` (AdamW(fused=True) over the unsharded mini-DDP), ``zero`` (ZeroRedundancyOptimizer with
AdamW(fused=True)) and ``overlap`` (the same with overlap_with_ddp=True).  Printed as JSON lines:

  * ``memory``: ``torch.cuda.max_memory_allocated`` over the timed steps, with W ranks sharing the one device (so the figure
    is the device's total for all W ranks), and at W = 1 the mean step time (backward + step, host-timed around device
    syncs).  Every configuration runs in a fresh process (nothing an earlier one left behind is counted), and the W = 1
    configurations are alternated and repeated ``--rounds`` times in this one job, so drift shows up as spread between
    rounds rather than as a difference between configurations;
  * ``kernel``: the W = 1 overlap kernel alone (k_local_step, AdamW, fp32 wire) over ``--launches`` launches on a
    ``--numel`` block, timed with CUDA events, and the bandwidth at its algorithmic bytes against the H100 SXM's 3.35 TB/s.

    python tools/zero_overlap_bench.py [--rounds 3] [--steps 4] [--batch 2] [--seq 1024]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

CONFIGS = ("unsharded", "zero", "overlap")
H100_HBM_BYTES_PER_S = 3.35e12


def alg_bytes_per_element(kind: str = "adamw") -> int:
    """Bytes the W = 1 fused pass moves per stepped fp32 element: the gradient read once (4 B), the parameter and the
    optimizer state read (4 B each) and written (4 B each).  Nothing else: the reduced gradient is not stored."""
    states = 2 if kind in ("adam", "adamw") else 1
    return 4 + 2 * 4 * (1 + states)


def measure(world: int, config: str, batch: int, seq: int, steps: int) -> dict:
    from zero_memory import gpt2

    from torchx_b200.ddp import Communicator, DistributedDataParallel, ZeroRedundancyOptimizer

    torch.cuda.empty_cache()
    if world > 1:  # load the broadcast's cat / copy kernels before the ranks wait on each other (see zero_memory.py)
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
                models.append(DistributedDataParallel(gpt2("cuda"), comms[r], broadcast_buffers=False,
                                                      algo="twoshot" if world > 1 else "auto"))
        torch.cuda.synchronize()
        for m in models:
            if config == "unsharded":
                opts.append(torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0.1, fused=True))
            else:
                opts.append(ZeroRedundancyOptimizer(m, torch.optim.AdamW, overlap_with_ddp=config == "overlap", lr=1e-4,
                                                    weight_decay=0.1, fused=True))
        g = torch.Generator().manual_seed(0)
        xs = [torch.randint(0, 50257, (batch, seq), generator=g).cuda() for _ in range(world)]

        def phase(fn):
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    fn(r)
            torch.cuda.synchronize()

        def loss(r):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return models[r](xs[r], labels=xs[r]).loss

        def backward(r):
            opts[r].zero_grad(set_to_none=True)
            loss(r).backward()

        def local_backward(r):  # loads every compute kernel with no collective in flight
            opts[r].zero_grad(set_to_none=True)
            with models[r].no_sync():
                loss(r).backward()
            opts[r].zero_grad(set_to_none=True)

        phase(local_backward)
        phase(backward)  # one untimed step: every kernel of the step is loaded
        phase(lambda r: opts[r].step())
        torch.cuda.reset_peak_memory_stats()
        times = []
        for _ in range(steps):
            t0 = time.perf_counter()
            phase(backward)
            phase(lambda r: opts[r].step())
            times.append(time.perf_counter() - t0)
        for c in comms:
            c.check()
        return {"world": world, "config": config, "batch": batch, "seq": seq,
                "max_memory_allocated_bytes": torch.cuda.max_memory_allocated(),
                "step_ms": round(1e3 * sum(times) / len(times), 2) if world == 1 else None}
    finally:
        del models, opts
        for c in comms:
            c.close()
        torch.cuda.synchronize()


def kernel(numel: int, launches: int) -> dict:
    """The W = 1 fused AdamW pass alone: one segment, one group, every element stepped."""
    from torchx_b200.ddp import Communicator
    from torchx_b200.ddp import _native as N

    (c,) = Communicator.create_local([0], stage_mb=8)
    try:
        grad = torch.randn(numel, device="cuda")
        p, m, v = torch.randn(numel, device="cuda"), torch.zeros(numel, device="cuda"), torch.zeros(numel, device="cuda")
        segs = (N.B2Segment * 1)()
        segs[0].src, segs[0].begin, segs[0].end = grad.data_ptr(), 0, numel
        t = N.B2Optim()
        t.kind, t.n_groups, t.n_runs = N.B2_OPT_ADAMW, 1, 1
        t.param, t.state0, t.state1 = p.data_ptr(), m.data_ptr(), v.data_ptr()
        t.run_begin[0], t.run_begin[1], t.run_group[0], t.run_step[0] = 0, numel, 0, 1.0
        g = t.group[0]
        g.lr, g.weight_decay, g.beta1, g.beta2, g.eps = 1e-4, 0.1, 0.9, 0.999, 1e-8
        for _ in range(3):
            c.reduce_scatter_step_(numel, segs, 1, t, scale=1.0, wire="f32")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            c.reduce_scatter_step_(numel, segs, 1, t, scale=1.0, wire="f32")
        e1.record()
        torch.cuda.synchronize()
        s = e0.elapsed_time(e1) * 1e-3 / launches
        b = alg_bytes_per_element("adamw") * numel
        return {"numel": numel, "launches": launches, "us_per_launch": round(s * 1e6, 2), "alg_bytes": b,
                "GB_per_s": round(b / s / 1e9, 1), "fraction_of_3.35_TB_per_s": round(b / s / H100_HBM_BYTES_PER_S, 3)}
    finally:
        c.close()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="repetitions of the alternated W = 1 configurations")
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--seq", type=int, default=1024)
    ap.add_argument("--worlds", type=int, nargs="*", default=[2, 4], help="worlds (one device) whose peaks are reported")
    ap.add_argument("--numel", type=int, default=1 << 25)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--one", nargs=2, metavar=("W", "CONFIG"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    if args.one:
        print(json.dumps(measure(int(args.one[0]), args.one[1], args.batch, args.seq, args.steps)), flush=True)
        return
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"kind": "device", "name": props.name}), flush=True)
    print(json.dumps({"kind": "kernel", **kernel(args.numel, args.launches)}), flush=True)
    runs = [(1, cfg, args.steps, rnd) for rnd in range(args.rounds)
            for cfg in (CONFIGS if rnd % 2 == 0 else CONFIGS[::-1])]  # alternate the order as well
    runs += [(w, cfg, 2, None) for w in args.worlds for cfg in CONFIGS]
    for w, cfg, steps, rnd in runs:
        # each configuration in a process of its own: the peak then counts nothing an earlier configuration left behind
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", str(w), cfg, "--steps", str(steps),
                              "--batch", str(args.batch), "--seq", str(args.seq)], capture_output=True, text=True, check=True)
        rec = json.loads(out.stdout.strip().splitlines()[-1])
        print(json.dumps({"kind": "memory", **({"round": rnd} if rnd is not None else {}), **rec}), flush=True)


if __name__ == "__main__":
    main()
