#!/usr/bin/env python
"""Where the time of bench.py's ResNet-50 step goes, per kernel group, and how close each BatchNorm pass comes to HBM.

    python tools/profile_resnet_step.py [--steps 5] [--warmup 5] [--tree DIR] [--out tool_out/profile_resnet_step]

Runs the bench's own step (``bench.Trainer``: B = 256, bf16 autocast, channels_last, SGD momentum, the mini-DDP at W = 1)
under ``torch.profiler`` with CUDA activities, after a warm-up, and reports:

* kernel time per step by group: ATen BatchNorm (its channels-last kernels), ours (``k_bn2d_*``), convolution / GEMM,
  ReLU / add / max-pool, optimizer, the bucket pass, other; the step time comes from a separate, unprofiled window timed
  with CUDA events;
* for every BatchNorm input shape [M = N*H*W, C]: the bytes an unfused BatchNorm must move (forward statistics read x,
  forward normalise read x + write y, backward reduce read x + dy, backward elementwise read x + dy + write dx: 8 passes
  of 2 B per element) over the measured time of those kernels, in GB/s and as a fraction of the H100 SXM data sheet's
  3.35 TB/s.  A layer whose ReLU runs inside its passes (``torchx_b200.nn.resnet``) moves more: its backward reduce also
  reads z and writes dy (+4 B per element), and its normalise reads the residual where it adds one (+2 B per element).

Kernels are matched to layers by their order within a step: forward kernels in module order, backward kernels in reverse.
``--tree DIR`` imports ``bench`` and ``torchx_b200`` from another checkout (a build of an earlier commit), so two versions
can be profiled by the same script.  The card's name, power limit and maximum SM clock (an ``nvidia-smi`` query) are
printed and written with the table to ``<out>.md`` and ``<out>.json``.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys

HBM_PEAK_GBS = 3350.0  # H100 SXM data sheet, HBM3

# (group, pattern on the kernel name); the first match wins
GROUPS = [
    ("ours_bn", re.compile(r"k_bn2d_")),
    ("aten_bn", re.compile(r"batch_norm")),
    ("bucket_pass", re.compile(r"\bk_(local_pass|oneshot|twoshot|pipe|ll)\b|k_local_pass")),
    ("optimizer", re.compile(r"multi_tensor_apply|foreach|sgd", re.I)),
    ("conv_gemm", re.compile(r"conv|xmma|implicit|gemm|cudnn|cutlass|wgrad|dgrad|fprop|nhwc|nchw|sm90_", re.I)),
    ("relu_add_pool", re.compile(r"clamp|relu|threshold|max_pool|AddFunctor|add_kernel|CUDAFunctor_add", re.I)),
]
# BatchNorm kernels -> (pass, bytes per element of x moved by that pass, direction)
BN_PASSES = [
    ("fwd_stats", re.compile(r"batch_norm_collect_statistics|k_bn2d_stats\b"), 1, "fwd"),
    ("fwd_norm", re.compile(r"batch_norm_transform_input|k_bn2d_norm\b"), 2, "fwd"),
    ("bwd_reduce", re.compile(r"batch_norm_backward_reduce|k_bn2d_bwd_reduce\b"), 2, "bwd"),
    ("bwd_elemt", re.compile(r"batch_norm_backward_elemt|k_bn2d_bwd_elemt\b"), 3, "bwd"),
]
# (pass, extra bytes per element of x) of a layer with the ReLU inside its passes, and of one that also adds the residual
FUSED_EXTRA = {"bwd_reduce": 4}
RESIDUAL_EXTRA = {"fwd_norm": 2}
# The small second launch of a native reduction whose tree spans several CTA rows (it folds their partials): its time
# belongs to the layer of the pass launched just before it
BN_TAILS = [
    ("fwd_stats", re.compile(r"k_bn2d_stats_merge\b")),
    ("bwd_reduce", re.compile(r"k_bn2d_bwd_reduce_merge\b")),
]


def group_of(name: str) -> str:
    for g, pat in GROUPS:
        if pat.search(name):
            return g
    return "other"


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": f"unknown ({type(e).__name__})", "power_limit": None, "sm_clock_max": None}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--timed-steps", type=int, default=20, help="unprofiled steps timed with CUDA events for the step time")
    ap.add_argument("--tree", default=None, help="import bench and torchx_b200 from this checkout")
    ap.add_argument("--out", default=os.path.join("tool_out", "profile_resnet_step"))
    args = ap.parse_args()
    root = os.path.abspath(args.tree) if args.tree else os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("profile_resnet_step.py needs a CUDA device")
    import bench

    targs = argparse.Namespace(model="resnet50", batch=256, impl="b200", wire="bf16", dump_outputs=None)
    tr = bench.Trainer(targs, 0, 1, 0)
    (xh, yh), = bench.synthetic_batches("resnet50", 256, 0, 1, pinned=False)
    x = xh.to(tr.device).contiguous(memory_format=torch.channels_last)
    y = yh.to(tr.device)

    # BatchNorm input shapes in forward order, from one hooked eval-mode forward (which leaves the running statistics alone),
    # and which layers a fused ResNet block (the class attributes of torchx_b200.nn.resnet's blocks) runs with their ReLU
    fused = {}
    for m in tr.ddp.module.modules():
        for name in getattr(type(m), "_fused_bns", ()):
            fused[id(getattr(m, name))] = "residual" if name == type(m)._residual_bn else "relu"
    shapes, kinds = [], []

    def record(m, i, o):
        shapes.append((i[0].shape[0] * i[0].shape[2] * i[0].shape[3], i[0].shape[1]))
        kinds.append(fused.get(id(m)))

    hooks = [m.register_forward_hook(record) for m in tr.ddp.module.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    tr.ddp.module.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        tr.ddp.module(x)
    tr.ddp.module.train()
    for h in hooks:
        h.remove()
    L = len(shapes)

    for _ in range(args.warmup):
        tr.step(x, y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.timed_steps):
        tr.step(x, y)
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / args.timed_steps

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            tr.step(x, y)
        torch.cuda.synchronize()
    kernels = sorted(((e.time_range.start, e.time_range.end - e.time_range.start, e.name) for e in prof.events()
                      if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name and "Memset" not in e.name),
                     key=lambda k: k[0])
    tr.close()

    per_group = collections.Counter()
    per_name = collections.Counter()
    for _, dur, name in kernels:
        per_group[group_of(name)] += dur
        per_name[name] += dur
    S = args.steps
    # BatchNorm kernels to layers: within each pass, occurrence k of a step is forward layer k or backward layer L-1-k
    per_shape = collections.defaultdict(lambda: collections.Counter())
    counts = collections.Counter()
    last_layer = {}
    for _, dur, name in kernels:
        for pname, pat, _, direction in BN_PASSES:
            if pat.search(name):
                k = counts[pname] % L
                counts[pname] += 1
                layer = k if direction == "fwd" else L - 1 - k
                per_shape[shapes[layer]][pname] += dur
                last_layer[pname] = layer
        for pname, pat in BN_TAILS:
            if pat.search(name) and pname in last_layer:
                per_shape[shapes[last_layer[pname]]][pname] += dur
    bn_launch_ok = all(counts[p] == S * L for p, *_ in BN_PASSES)

    info = card()
    total_us = sum(per_group.values()) / S
    rows = []
    for (M, C) in sorted(set(shapes), key=lambda s: -s[0] * s[1]):
        layers = [kinds[k] for k in range(L) if shapes[k] == (M, C)]
        nl = len(layers)
        t = per_shape[(M, C)]
        row = {"M": M, "C": C, "layers": nl, "fused_layers": sum(1 for k in layers if k), "MiB_bf16": round(M * C * 2 / 2**20, 1)}
        tot_b, tot_t = 0, 0.0
        for pname, _, bpe, _ in BN_PASSES:
            us = t[pname] / S
            b = sum(bpe * 2 + (FUSED_EXTRA.get(pname, 0) if k else 0) + (RESIDUAL_EXTRA.get(pname, 0) if k == "residual" else 0)
                    for k in layers) * M * C
            row[pname + "_us"] = round(us, 1)
            row[pname + "_gbs"] = round(b / (us * 1e-6) / 1e9, 1) if us > 0 else None
            tot_b += b
            tot_t += us
        row["all_gbs"] = round(tot_b / (tot_t * 1e-6) / 1e9, 1) if tot_t > 0 else None
        row["all_frac"] = round(tot_b / (tot_t * 1e-6) / 1e9 / HBM_PEAK_GBS, 3) if tot_t > 0 else None
        rows.append(row)
    res = {
        "card": info, "tree": root, "steps_profiled": S, "step_ms": round(step_ms, 3), "kernel_ms_per_step": round(total_us / 1e3, 3),
        "groups_ms_per_step": {g: round(v / S / 1e3, 3) for g, v in per_group.most_common()},
        "groups_share_of_step": {g: round(v / S / 1e3 / step_ms, 4) for g, v in per_group.most_common()},
        "bn_layers": L, "bn_kernels_matched": bn_launch_ok, "bn_shapes": rows,
        "top_kernels_ms_per_step": [(n[:160], round(v / S / 1e3, 3)) for n, v in per_name.most_common(25)],
    }
    lines = [f"# ResNet-50 step profile ({root})", "",
             f"Card: {info['name']}, power limit {info['power_limit']}, max SM clock {info['sm_clock_max']}.",
             f"Step time (CUDA events, {args.timed_steps} unprofiled steps): {step_ms:.2f} ms.  Kernel time per step (profiled, "
             f"{S} steps): {total_us / 1e3:.2f} ms.", "",
             "| group | ms / step | share of step |", "|---|---:|---:|"]
    for g, v in per_group.most_common():
        lines.append(f"| {g} | {v / S / 1e3:.2f} | {v / S / 1e3 / step_ms:.1%} |")
    lines += ["", f"BatchNorm layers: {L}; every pass matched S x L kernels: {bn_launch_ok}.", "",
              "| M | C | layers | fused | MiB bf16 | fwd stats GB/s | fwd norm GB/s | bwd reduce GB/s | bwd elemt GB/s | all passes GB/s | of 3.35 TB/s |",
              "|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|"]
    for r in rows:
        lines.append(f"| {r['M']} | {r['C']} | {r['layers']} | {r['fused_layers']} | {r['MiB_bf16']} | {r['fwd_stats_gbs']} | {r['fwd_norm_gbs']} | "
                     f"{r['bwd_reduce_gbs']} | {r['bwd_elemt_gbs']} | {r['all_gbs']} | {r['all_frac']} |")
    lines += ["", "| kernel | ms / step |", "|---|---:|"] + [f"| `{n}` | {v} |" for n, v in res["top_kernels_ms_per_step"]]
    text = "\n".join(lines) + "\n"
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out + ".md", "w") as f:
        f.write(text)
    with open(args.out + ".json", "w") as f:
        json.dump(res, f, indent=1)
    print(text)


if __name__ == "__main__":
    main()
