"""Generates the fp16 golden fixtures by RUNNING THE REFERENCE (a checkout of meta-pytorch/torchx, named by the
TORCHX_REFERENCE environment variable), the same way make_golden.py makes ddp_w{2,4}.npz:

  ddp_fp16_w{2,4}.npz   stock torch DistributedDataParallel launched through the reference's own launcher
                        (PYTHONPATH=$TORCHX_REFERENCE python -m torchx.cli.main run -s local_cwd
                        $TORCHX_REFERENCE/torchx/components/dist.py:ddp -j 1xW --script <worker>, gloo on CPU):
                          local_f32 / ddp_fp16_compress   fp32 model, default_hooks.fp16_compress_hook
                          local_f16 / ddp_f16_none        the same model .half(), no hook (fp16 bucket, pre-divide, SUM)
                        local_* hold every rank's own gradients (fp16 ones as uint16 bits), ddp_* every rank's result.

Run from the repo root:  python tests/golden/make_golden_fp16.py      (needs TORCHX_REFERENCE; not needed at test time)
"""
import os
import subprocess
import sys
import tempfile
import textwrap

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("TORCHX_REFERENCE", "")

WORKER = textwrap.dedent(
    '''
    import argparse
    import numpy as np
    import torch, torch.nn as nn, torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP
    from torch.distributed.algorithms.ddp_comm_hooks import default_hooks

    ap = argparse.ArgumentParser(); ap.add_argument("--out"); a = ap.parse_args()
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()

    def model(half):
        torch.manual_seed(0)
        m = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 16))
        return m.half() if half else m

    torch.manual_seed(100 + rank)
    x = torch.randn(32, 64)

    def flat_grads(m):
        return torch.cat([p.grad.reshape(-1) for p in m.parameters()])

    def gather(v):
        g = [torch.empty_like(v) for _ in range(world)]
        dist.all_gather(g, v)
        return torch.stack(g)

    def bits(t):
        return t.view(torch.int16).numpy().view(np.uint16) if t.dtype == torch.float16 else t.numpy()

    out = {}
    for half, tag in ((False, "f32"), (True, "f16")):
        xin = x.half() if half else x
        m = model(half); m(xin).float().sum().backward()
        out["local_" + tag] = bits(gather(flat_grads(m).clone()))
    for name, half, hook in (("fp16_compress", False, default_hooks.fp16_compress_hook), ("f16_none", True, None)):
        d = DDP(model(half))
        if hook is not None:
            d.register_comm_hook(None, hook)
        d(x.half() if half else x).float().sum().backward()
        out["ddp_" + name] = bits(gather(flat_grads(d.module).clone()))
        dist.barrier()
    if rank == 0:
        np.savez(a.out, **out)
    dist.barrier()
    dist.destroy_process_group()
    '''
)


def run_reference_ddp_fp16(world: int) -> None:
    out = os.path.join(HERE, f"ddp_fp16_w{world}.npz")
    with tempfile.TemporaryDirectory() as td:
        script = os.path.join(td, "golden_fp16_worker.py")
        with open(script, "w") as f:
            f.write(WORKER)
        env = dict(os.environ, PYTHONPATH=REF)
        cmd = [sys.executable, "-m", "torchx.cli.main", "run", "-s", "local_cwd", f"{REF}/torchx/components/dist.py:ddp",
               "-j", f"1x{world}", "--script", script, "--", "--out", out]
        subprocess.run(cmd, check=True, cwd=td, env=env)
    assert os.path.exists(out), out
    print("wrote", out)


if __name__ == "__main__":
    if not os.path.isdir(os.path.join(REF, "torchx")):
        raise SystemExit(f"TORCHX_REFERENCE={REF!r} is not a checkout of meta-pytorch/torchx (no torchx/ package in it); "
                         "set it to regenerate the fp16 ddp fixtures")
    for w in (2, 4):
        run_reference_ddp_fp16(w)
