"""ZeRO-1 with fp32 master weights for a bf16 model (``master_weights=True``) against fp32 parameters, GPT-2-small,
AdamW(fused=True), both with the step inside the backward's reduce-scatter (``overlap_with_ddp=True``).

Three parts, printed as JSON lines:

  * ``state_bytes`` (no GPU, ``--cpu-only``): the exact bytes each rank keeps between steps at W = 1, 2 and 4, from the
    parameter shapes and the mini-DDP's default bucket plan.  A rank keeps every bucket's flat parameter buffer (W * block
    elements of the parameter dtype), and for each bucket ``block`` fp32 elements of exp_avg and of exp_avg_sq, plus
    ``block`` fp32 masters for a bf16 bucket;
  * ``memory``: ``torch.cuda.max_memory_allocated`` over ``--steps`` steps with W ranks sharing the one device (so the
    figure is the device's total for all W ranks), each configuration in a fresh process.  ``fp32`` trains the fp32 model
    under bf16 autocast, ``bf16_masters`` the ``model.bfloat16()`` model without autocast;
  * ``kernel``: the W = 1 fused AdamW pass (k_local_step) on a ``--numel`` block, its bf16 instance (bf16 gradient,
    fp32 master and state, bf16 parameter written) and its fp32 instance (fp32 wire) alternated over ``--rounds`` rounds of
    ``--launches`` launches, timed with CUDA events.

    python tools/zero_master_bench.py --cpu-only
    python tools/zero_master_bench.py [--steps 3] [--batch 2] [--seq 1024] [--numel 33554432] [--launches 200]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from typing import Sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

WORLDS = (1, 2, 4)
CONFIGS = ("fp32", "bf16_masters")
H100_HBM_BYTES_PER_S = 3.35e12


def alg_bytes_per_element(master: bool) -> int:
    """Bytes the W = 1 fused AdamW pass moves per stepped element.  fp32: the gradient read (4 B), the parameter, exp_avg
    and exp_avg_sq read and written (24 B).  bf16 with a master: the bf16 gradient read (2 B), the master and the two
    states read and written (24 B), the bf16 parameter written (2 B)."""
    return 2 + 24 + 2 if master else 4 + 24


def bytes_per_rank(numels: Sequence[int], elem_bytes: int, world: int, masters: bool) -> dict:
    """Exact bytes one rank keeps between steps for parameters of ``numels`` elements of ``elem_bytes`` bytes each, with
    AdamW in the overlap mode and the default bucket plan (1 MiB first bucket, 25 MiB buckets)."""
    from torchx_b200.ddp.bucketing import MIB, plan_buckets
    from torchx_b200.ddp.zero import padded_block

    dtype = {4: "torch.float32", 2: "torch.bfloat16"}[elem_bytes]
    specs = plan_buckets(list(numels), [elem_bytes] * len(numels), [dtype] * len(numels), 1 * MIB, 25 * MIB)
    blocks = [padded_block(s.numel, world) for s in specs]
    params = sum(world * b for b in blocks) * elem_bytes
    state = sum(blocks) * 8
    master = sum(blocks) * 4 if masters else 0
    return {"world": world, "params": sum(numels), "param_bytes": params, "state_bytes": state, "master_bytes": master,
            "total_bytes": params + state + master}


def state_bytes(world: int) -> dict:
    from zero_memory import gpt2

    numels = [p.numel() for p in gpt2("meta").parameters() if p.requires_grad]
    return {"kind": "state_bytes", "fp32": bytes_per_rank(numels, 4, world, False),
            "bf16_masters": bytes_per_rank(numels, 2, world, True)}


def measure(world: int, config: str, batch: int, seq: int, steps: int) -> dict:
    from zero_memory import gpt2

    from torchx_b200.ddp import Communicator, DistributedDataParallel, ZeroRedundancyOptimizer

    bf16 = config == "bf16_masters"

    def model():
        m = gpt2("cuda")
        return m.bfloat16() if bf16 else m

    torch.cuda.empty_cache()
    if world > 1:  # load the broadcast's cat / copy kernels before the ranks wait on each other (see zero_memory.py)
        import types

        stub = types.SimpleNamespace(world_size=world, comm=types.SimpleNamespace(rank=1, broadcast_=lambda t, root: t))
        m = model()
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
                models.append(DistributedDataParallel(model(), comms[r], broadcast_buffers=False,
                                                      algo="twoshot" if world > 1 else "auto"))
        torch.cuda.synchronize()
        for m in models:
            opts.append(ZeroRedundancyOptimizer(m, torch.optim.AdamW, overlap_with_ddp=True, master_weights=bf16, lr=1e-4,
                                                weight_decay=0.1, fused=True))
        g = torch.Generator().manual_seed(0)
        xs = [torch.randint(0, 50257, (batch, seq), generator=g).cuda() for _ in range(world)]

        def phase(fn):
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    fn(r)
            torch.cuda.synchronize()

        def loss(r):
            if bf16:
                return models[r](xs[r], labels=xs[r]).loss
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
        phase(backward)
        phase(lambda r: opts[r].step())
        torch.cuda.reset_peak_memory_stats()
        for _ in range(steps):
            phase(backward)
            phase(lambda r: opts[r].step())
        for c in comms:
            c.check()
        return {"world": world, "config": config, "batch": batch, "seq": seq,
                "max_memory_allocated_bytes": torch.cuda.max_memory_allocated()}
    finally:
        del models, opts
        for c in comms:
            c.close()
        torch.cuda.synchronize()


def kernel(numel: int, launches: int, rounds: int) -> dict:
    """The W = 1 fused AdamW pass alone, bf16 instance against fp32 instance: one segment, one group, every element stepped."""
    from torchx_b200.ddp import Communicator
    from torchx_b200.ddp import _native as N

    (c,) = Communicator.create_local([0], stage_mb=8)
    try:
        gen = torch.Generator(device="cuda").manual_seed(0)
        g32 = torch.randn(numel, device="cuda", generator=gen)
        g16 = g32.bfloat16()
        p32, m32, v32 = torch.randn(numel, device="cuda", generator=gen), torch.zeros(numel, device="cuda"), torch.zeros(numel, device="cuda")
        master, m16, v16 = p32.clone(), torch.zeros(numel, device="cuda"), torch.zeros(numel, device="cuda")
        pbf = master.bfloat16()

        def table(grad, param, m, v):
            segs = (N.B2Segment * 1)()
            segs[0].src, segs[0].begin, segs[0].end = grad.data_ptr(), 0, numel
            t = N.B2Optim()
            t.kind, t.n_groups, t.n_runs = N.B2_OPT_ADAMW, 1, 1
            t.param, t.state0, t.state1 = param.data_ptr(), m.data_ptr(), v.data_ptr()
            t.run_begin[0], t.run_begin[1], t.run_group[0], t.run_step[0] = 0, numel, 0, 1.0
            h = t.group[0]
            h.lr, h.weight_decay, h.beta1, h.beta2, h.eps = 1e-4, 0.1, 0.9, 0.999, 1e-8
            return segs, t

        s32, t32 = table(g32, p32, m32, v32)
        s16, t16 = table(g16, master, m16, v16)
        run = {"fp32": lambda: c.reduce_scatter_step_(numel, s32, 1, t32, scale=1.0, wire="f32"),
               "bf16_master": lambda: c.reduce_scatter_step_bf16_(numel, s16, 1, t16, pbf, scale=1.0)}
        for f in run.values():
            for _ in range(3):
                f()
        times = {k: [] for k in run}
        for rnd in range(rounds):
            for k in (list(run) if rnd % 2 == 0 else list(run)[::-1]):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(launches):
                    run[k]()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e-3 / launches)
        c.check()
        out = {"numel": numel, "launches": launches, "rounds": rounds}
        for k, ts in times.items():
            b = alg_bytes_per_element(k == "bf16_master") * numel
            s = sorted(ts)[len(ts) // 2]
            out[k] = {"us_per_launch_median": round(s * 1e6, 2), "us_per_launch_all": [round(t * 1e6, 2) for t in ts],
                      "alg_bytes": b, "GB_per_s": round(b / s / 1e9, 1), "fraction_of_3.35_TB_per_s": round(b / s / H100_HBM_BYTES_PER_S, 3)}
        return out
    finally:
        c.close()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpu-only", action="store_true", help="only the exact bytes per rank (no GPU)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--seq", type=int, default=1024)
    ap.add_argument("--numel", type=int, default=1 << 25)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--one", nargs=2, metavar=("W", "CONFIG"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.one:
        os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
        print(json.dumps(measure(int(args.one[0]), args.one[1], args.batch, args.seq, args.steps)), flush=True)
        return
    for w in WORLDS:
        print(json.dumps(state_bytes(w)), flush=True)
    if args.cpu_only:
        return
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"kind": "device", "name": torch.cuda.get_device_name(0), "nvidia_smi": smi[:1]}), flush=True)
    print(json.dumps({"kind": "kernel", **kernel(args.numel, args.launches, args.rounds)}), flush=True)
    for w in WORLDS:
        for cfg in CONFIGS:
            # each configuration in a process of its own: the peak then counts nothing an earlier one left behind
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", str(w), cfg, "--steps", str(args.steps),
                                  "--batch", str(args.batch), "--seq", str(args.seq)], capture_output=True, text=True, check=True)
            print(json.dumps({"kind": "memory", **json.loads(out.stdout.strip().splitlines()[-1])}), flush=True)


if __name__ == "__main__":
    main()
