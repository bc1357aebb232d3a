#!/usr/bin/env python
"""bench.py's ResNet-50 step with the model converted to SyncBatchNorm, under init_pg("b200") and the mini-DDP.

    python tools/syncbn_resnet_bench.py [--trees DIR,DIR] [--rounds 3] [--steps 50] [--warmup 10] [--profile-steps 5]
                                        [--world-check 2] [--out tool_out/syncbn_resnet_bench]

The step is ``bench.Trainer.step``'s: B = 256 per rank, bf16 autocast, channels_last, SGD with momentum, the model from
``bench.build_model("resnet50")`` passed through ``torchx_b200.nn.SyncBatchNorm.convert_sync_batchnorm`` and wrapped by the
mini-DDP at W = 1 (so every SyncBatchNorm layer runs its one-rank path).  Each tree of ``--trees`` (checkouts with a built
library, e.g. an earlier commit's and this one) is run in a fresh process per round, the trees alternating, for
``--rounds`` rounds: images/s from CUDA events over ``--steps`` steps after ``--warmup``.  The last round also profiles
``--profile-steps`` steps under ``torch.profiler`` and reports kernel time per step in ``tools/profile_resnet_step.py``'s
groups (ATen BatchNorm, the native ``k_bn2d_*`` kernels, ReLU / add / max-pool, ...).  ``--world-check W`` then runs a few
steps of the same training at W ranks sharing device 0 with every tree and reports only that they complete: time-sliced
ranks measure nothing about NVLink.  The card's name, power limit and maximum SM clock are read in the same run, and
each timed round records the SM clock the card runs at (``nvidia-smi --query-gpu=clocks.sm``) right after its timed steps.
"""
import argparse
import json
import os
import subprocess
import sys
import uuid

TOOLS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TOOLS)


def sm_clock() -> str:
    """The current SM clock of device 0 (a read-only nvidia-smi query), or "unknown"."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({type(e).__name__})"


def child(a) -> None:
    tree = os.path.abspath(a.tree)
    sys.path.insert(0, tree)
    sys.path.insert(1, TOOLS)
    os.environ.update(RANK=str(a.rank), WORLD_SIZE=str(a.world), LOCAL_RANK=str(a.rank), B2_DEVICE="0", B2_SHM_NAME=a.shm)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("syncbn_resnet_bench.py needs a CUDA device")
    import bench
    import profile_resnet_step as P
    import torchx_b200.distributed as D
    from torchx_b200.ddp import DistributedDataParallel
    from torchx_b200.nn import SyncBatchNorm

    assert os.path.dirname(os.path.abspath(bench.__file__)) == tree
    device = D.init_pg("b200")
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    model = SyncBatchNorm.convert_sync_batchnorm(bench.build_model("resnet50", device))
    ddp = DistributedDataParallel(model, D.communicator(), wire="bf16")
    opt = torch.optim.SGD(ddp.parameters(), lr=0.1, momentum=0.9)
    loss_fn = torch.nn.CrossEntropyLoss()
    (xh, yh), = bench.synthetic_batches("resnet50", a.batch, a.rank, 1, pinned=False)
    x = xh.to(device).contiguous(memory_format=torch.channels_last)
    y = yh.to(device)

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = loss_fn(ddp(x), y)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        return loss

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    res = {"tree": tree, "world": a.world, "rank": a.rank, "ms_per_step": round(ms, 3),
           "images_per_s": round(a.batch * a.world / (ms / 1e3), 1), "loss": float(loss), "sm_clock_after_timed_steps": sm_clock()}
    if a.profile_steps:
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_steps):
                step()
            torch.cuda.synchronize()
        groups = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name and "Memset" not in e.name:
                g = P.group_of(e.name)
                groups[g] = groups.get(g, 0.0) + (e.time_range.end - e.time_range.start)
        res["kernel_ms_per_step"] = {g: round(v / a.profile_steps / 1e3, 3) for g, v in sorted(groups.items(), key=lambda kv: -kv[1])}
    D.barrier()
    D.communicator().close()
    print("RESULT " + json.dumps(res), flush=True)


def run(tree, world, a, steps, warmup, profile_steps):
    shm = f"/b2_sbnb_{uuid.uuid4().hex[:12]}"
    cmd = [sys.executable, os.path.abspath(__file__), "--child", "--tree", tree, "--world", str(world), "--shm", shm, "--batch",
           str(a.batch), "--steps", str(steps), "--warmup", str(warmup), "--profile-steps", str(profile_steps)]
    procs = []
    try:
        for r in range(world):
            procs.append(subprocess.Popen(cmd + ["--rank", str(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
        outs = [p.communicate(timeout=3600)[0] for p in procs]
    finally:  # a rank that failed or hung leaves no process behind on the shared GPU
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    for p, o in zip(procs, outs):
        if p.returncode != 0:
            raise SystemExit(f"{tree} W={world} failed:\n{o}")
    return [json.loads(line[len("RESULT "):]) for o in outs for line in o.splitlines() if line.startswith("RESULT ")]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", default=ROOT, help="comma-separated checkouts, each with a built library")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--world-check", type=int, default=2, help="then run a few steps at this many ranks sharing device 0 (0: skip)")
    ap.add_argument("--out", default=os.path.join("tool_out", "syncbn_resnet_bench"))
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--tree", help=argparse.SUPPRESS)
    ap.add_argument("--rank", type=int, default=0, help=argparse.SUPPRESS)
    ap.add_argument("--world", type=int, default=1, help=argparse.SUPPRESS)
    ap.add_argument("--shm", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a)
    sys.path.insert(0, TOOLS)
    import profile_resnet_step as P

    trees = [os.path.abspath(t) for t in a.trees.split(",")]
    out = {"card": P.card(), "batch": a.batch, "steps": a.steps, "warmup": a.warmup, "rounds": []}
    for r in range(a.rounds):
        for t in trees:
            res = run(t, 1, a, a.steps, a.warmup, a.profile_steps if r == a.rounds - 1 else 0)[0]
            out["rounds"].append(res)
            print(json.dumps(res), flush=True)
    if a.world_check > 1:
        out["world_check"] = []
        for t in trees:
            res = run(t, a.world_check, a, 3, 2, 0)
            out["world_check"].append({"tree": t, "world": a.world_check, "completed": len(res) == a.world_check,
                                       "losses": [x["loss"] for x in res]})
            print(json.dumps(out["world_check"][-1]), flush=True)
    out["card_after"] = P.card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out + ".json", "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"card": out["card"], "card_after": out["card_after"]}))


if __name__ == "__main__":
    main()
