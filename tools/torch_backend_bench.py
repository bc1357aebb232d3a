"""What the "b200" torch.distributed backend costs on one GPU (W = 1).

  * bench.py's ResNet-50 step (bf16 autocast, channels_last, B = 256, SGD momentum) under stock torch DDP on a "b200"
    group, the same under stock DDP on an NCCL group, and under the mini-DDP: images/s, in alternated rounds;
  * host time per ``dist.all_reduce`` of one element through the Python process group, against ``D.all_reduce`` on the
    fabric with no group (and NCCL's for scale).

    python tools/torch_backend_bench.py [--rounds 3] [--steps 20] [--warmup 5] [--out result.json]

Prints one JSON object with the GPU's name, power limit and the SM clocks seen before and after.  Multi-GPU throughput
is not measured here.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import time
import uuid

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    os.environ.update(RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", B2_DEVICE="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                      B2_SHM_NAME=f"/b2_tbb_{uuid.uuid4().hex[:12]}")

    import torch
    import torch.distributed as dist
    import torchvision
    from torch.nn.parallel import DistributedDataParallel as TorchDDP

    import torchx_b200.distributed as D
    from torchx_b200.ddp import DistributedDataParallel

    assert torch.cuda.is_available(), "torch_backend_bench needs a CUDA device"
    before = gpu_info()
    dev = D.init_pg("b200")
    g = torch.Generator().manual_seed(1000)
    x = torch.randn(a.batch, 3, 224, 224, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (a.batch,), generator=g).to(dev)
    loss_fn = torch.nn.CrossEntropyLoss()

    def resnet_rate(arm):
        if arm in ("b200", "nccl"):
            dist.init_process_group(arm, device_id=None if arm == "b200" else dev)
        torch.manual_seed(0)
        model = torchvision.models.resnet50().to(dev).to(memory_format=torch.channels_last)
        ddp = TorchDDP(model, device_ids=[dev.index]) if arm != "mini" else DistributedDataParallel(model)
        opt = torch.optim.SGD(ddp.parameters(), lr=0.1, momentum=0.9)

        def step():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = loss_fn(ddp(x), y)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()

        for _ in range(a.warmup):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        del ddp, opt, model
        if arm in ("b200", "nccl"):
            dist.destroy_process_group()
        return a.steps * a.batch / (ms / 1e3)

    def host_us(arm):
        if arm in ("b200", "nccl"):
            dist.init_process_group(arm, device_id=None if arm == "b200" else dev)
        t = torch.zeros(1, device=dev)
        fn = D.all_reduce if arm == "fabric" else dist.all_reduce
        for _ in range(50):
            fn(t)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.calls):
            fn(t)
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        if arm in ("b200", "nccl"):
            dist.destroy_process_group()
        return {"enqueue_us": (t1 - t0) / a.calls * 1e6, "with_sync_us": (t2 - t0) / a.calls * 1e6}

    rates = {"b200": [], "nccl": [], "mini": []}
    calls = {"fabric": [], "b200": [], "nccl": []}
    for _ in range(a.rounds):
        for arm in rates:
            rates[arm].append(resnet_rate(arm))
        for arm in calls:
            calls[arm].append(host_us(arm))
    after = gpu_info()
    result = {
        "gpu_before": before, "gpu_after": after, "world": 1, "batch": a.batch, "steps": a.steps, "warmup": a.warmup,
        "resnet50_images_per_s": {k: [round(v, 1) for v in vs] for k, vs in rates.items()},
        "allreduce_1_elem_host_us": {k: [{m: round(u, 2) for m, u in v.items()} for v in vs] for k, vs in calls.items()},
    }
    line = json.dumps(result)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    D.communicator().close()


if __name__ == "__main__":
    main()
