#!/usr/bin/env python
"""What find_unused_parameters=True costs the mini-DDP on bench.py's workload: ResNet-50, B=256 per GPU, 3x224x224,
channels_last, bf16 autocast, SGD with momentum, at W = 1.  Two mini-DDPs over identical models, one with the flag off
and one with it on, are timed in alternating rounds (device events around `--steps` steps after `--warmup` steps).  The
host time of the graph walk that finds the unused parameters (the output walk plus the autograd graph walk of one
forward) is timed on its own after the rounds.  Prints one JSON line; with --out it is also written there.

    python tools/unused_params_overhead.py --steps 20 --warmup 5 --rounds 2

The walk is host work at every synced forward; at W > 1 the flag also adds one MAX reduction of an int32 map per synced
backward and, when some parameter is unused on this rank, a host wait for it in the backward's final callback."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--walks", type=int, default=20, help="forwards whose graph walk is timed on its own")
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import torch
    import torchvision

    from torchx_b200.ddp import Communicator, DistributedDataParallel
    from torchx_b200.ddp.ddp import _find_tensors, _reached_leaves

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cudnn.benchmark = True
    comm = Communicator.create(0, 1, 0, "/unused", stage_mb=8)
    arms = {}
    for flag in (False, True):
        torch.manual_seed(0)
        model = torchvision.models.resnet50().to(dev).to(memory_format=torch.channels_last)
        ddp = DistributedDataParallel(model, comm, find_unused_parameters=flag)
        arms[flag] = (ddp, torch.optim.SGD(ddp.parameters(), lr=0.1, momentum=0.9))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(a.batch, 3, 224, 224, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (a.batch,), generator=g).to(dev)
    loss_fn = torch.nn.CrossEntropyLoss()

    def step(ddp, opt):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = loss_fn(ddp(x), y)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    times = {False: [], True: []}
    for _ in range(a.rounds):
        for flag in (False, True):
            ddp, opt = arms[flag]
            for _ in range(a.warmup):
                step(ddp, opt)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                step(ddp, opt)
            e1.record()
            torch.cuda.synchronize()
            times[flag].append(e0.elapsed_time(e1) / a.steps)
    ddp, opt = arms[True]
    walk_ms, nodes_reached = [], 0
    for _ in range(a.walks):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = ddp.module(x)
        t0 = time.perf_counter()
        reached = _reached_leaves(_find_tensors(out))
        walk_ms.append((time.perf_counter() - t0) * 1e3)
        nodes_reached = len(reached)
        del out
    torch.cuda.synchronize()
    comm.close()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        card = "unknown"
    line = {
        "workload": f"ResNet-50 mini-DDP W=1, B={a.batch}, 3x224x224, channels_last, bf16 autocast, SGD momentum",
        "gpu": card,
        "step_ms_find_unused_false": [round(t, 3) for t in times[False]],
        "step_ms_find_unused_true": [round(t, 3) for t in times[True]],
        "images_per_s_false": round(a.batch * 1e3 / statistics.mean(times[False]), 1),
        "images_per_s_true": round(a.batch * 1e3 / statistics.mean(times[True]), 1),
        "graph_walk_ms_median": round(statistics.median(walk_ms), 3),
        "graph_walk_ms_max": round(max(walk_ms), 3),
        "parameters_reached": nodes_reached,
        "parameters_trainable": len(ddp._params),
    }
    s = json.dumps(line)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
