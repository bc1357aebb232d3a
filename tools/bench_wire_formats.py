#!/usr/bin/env python
"""Single-H100 comparison of the five wire formats (B2_* modes 0..4), one call, CUDA events only:

  1. the fused cast/scale pass (b2_local_pass, the W = 1 bucket kernel) in every mode over bucket sizes from 1 MiB to
     1 GiB, the modes interleaved round by round so that clock and thermal drift hit all of them alike; GB/s at the
     algorithmic bytes (read the bucket once, write it once: 8 B per element for fp32 buckets, 4 B for 16-bit ones)
     against the 3.35 TB/s HBM3 data-sheet figure;
  2. a ResNet-50 training step through the mini-DDP on one GPU: fp16 autocast + GradScaler + wire="f16" against bf16
     autocast + wire="bf16", interleaved.

Prints one JSON line per measurement and a header line with the card's name and power limit, which are part of every
number here.  Multi-GPU timing is out of its scope.

    python tools/bench_wire_formats.py [--sizes-mib 1,4,16,64,256,1024] [--rounds 5] [--resnet-steps 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from torchx_b200.ddp import _native as N  # noqa: E402
from torchx_b200.ddp import local_pass_  # noqa: E402

HBM_GBS = 3350.0  # H100 SXM HBM3 data-sheet bandwidth
# mode -> (bucket dtype, wire= argument)
MODES = {
    "f32_wire_bf16": (torch.float32, "bf16"),
    "f32": (torch.float32, "f32"),
    "bf16": (torch.bfloat16, "bf16"),
    "f32_wire_f16": (torch.float32, "f16"),
    "f16": (torch.float16, "f16"),
}


def card() -> dict:
    p = torch.cuda.get_device_properties(0)
    info = {"gpu": p.name, "sms": p.multi_processor_count}
    try:  # read-only query
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception as e:  # noqa: BLE001
        info["power_limit_w"] = None
        info["power_limit_error"] = str(e)[:200]
    return info


def time_pass(bufs, wire, iters) -> float:
    for b in bufs[:2]:
        local_pass_(b, scale=1.0, wire=wire)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for i in range(iters):
        local_pass_(bufs[i % len(bufs)], scale=1.0, wire=wire)
    ev1.record()
    ev1.synchronize()
    return ev0.elapsed_time(ev1) * 1e-3 / iters


def local_pass_sweep(sizes_mib, rounds):
    for mib in sizes_mib:
        nbytes = int(mib * (1 << 20))
        bufs, iters = {}, max(5, min(50, int(2e10 / nbytes)))
        for name, (dt, _) in MODES.items():
            n = nbytes // torch.tensor([], dtype=dt).element_size()
            nbuf = max(1, min(16, (512 << 20) // nbytes + 1))  # rotate through > 50 MB of L2
            bufs[name] = [torch.randn(n, device="cuda:0").to(dt) for _ in range(nbuf)]
        times = {name: [] for name in MODES}
        for _ in range(rounds):
            for name, (_, wire) in MODES.items():
                times[name].append(time_pass(bufs[name], wire, iters))
        for name, (dt, wire) in MODES.items():
            n = bufs[name][0].numel()
            t = statistics.median(times[name])
            alg = 2 * n * bufs[name][0].element_size()
            print(json.dumps({"bench": "local_pass", "mode": name, "bucket_mib": mib, "n": n, "us_median": round(t * 1e6, 2),
                              "us_min": round(min(times[name]) * 1e6, 2), "gbs": round(alg / t / 1e9, 1),
                              "frac_of_hbm": round(alg / t / 1e9 / HBM_GBS, 3), "rounds": rounds, "iters": iters}), flush=True)
        del bufs
        torch.cuda.empty_cache()


def resnet_steps(steps, rounds, batch):
    import torchvision

    from torchx_b200.ddp import Communicator, DistributedDataParallel

    comm = Communicator.create_local([0], stage_mb=8)[0]
    torch.manual_seed(0)
    x = torch.randn(batch, 3, 224, 224, device="cuda:0").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device="cuda:0")
    setups = {}
    for name, dt, wire in (("fp16_autocast_gradscaler_wire_f16", torch.float16, "f16"), ("bf16_autocast_wire_bf16", torch.bfloat16, "bf16")):
        m = torchvision.models.resnet50().cuda().to(memory_format=torch.channels_last)
        d = DistributedDataParallel(m, comm, wire=wire)
        opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9)
        scaler = torch.amp.GradScaler("cuda") if dt == torch.float16 else None
        setups[name] = (d, opt, scaler, dt)

    def step(d, opt, scaler, dt):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=dt):
            loss = torch.nn.functional.cross_entropy(d(x), y)
        if scaler is None:
            loss.backward()
            opt.step()
        else:
            scaler.scale(loss).backward()
            scaler.step(opt)
            scaler.update()

    for s in setups.values():
        for _ in range(3):
            step(*s)
    torch.cuda.synchronize()
    times = {name: [] for name in setups}
    for _ in range(rounds):
        for name, s in setups.items():
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(steps):
                step(*s)
            ev1.record()
            ev1.synchronize()
            times[name].append(ev0.elapsed_time(ev1) * 1e-3 / steps)
    for name in setups:
        t = statistics.median(times[name])
        print(json.dumps({"bench": "resnet50_step_1gpu", "config": name, "batch": batch, "ms_median": round(t * 1e3, 2),
                          "images_per_s": round(batch / t, 1), "rounds": rounds, "steps_per_round": steps}), flush=True)
    comm.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes-mib", default="1,4,16,64,256,1024")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--resnet-steps", type=int, default=20)
    ap.add_argument("--resnet-rounds", type=int, default=4)
    ap.add_argument("--batch", type=int, default=128)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    print(json.dumps({"bench": "header", **card(), "abi": N.lib().b2_version(), "hbm_gbs_datasheet": HBM_GBS}), flush=True)
    local_pass_sweep([float(s) for s in a.sizes_mib.split(",")], a.rounds)
    if a.resnet_steps > 0:
        resnet_steps(a.resnet_steps, a.resnet_rounds, a.batch)


if __name__ == "__main__":
    main()
