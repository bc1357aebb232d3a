"""One rank of a multi-process topology (spawned by tests/test_ipc_gpu.py). Exercises the real rendezvous:
POSIX-shm control block + arena exchange (VMM file descriptors + NVSwitch multicast where the box offers them, else
CUDA IPC), then allreduce / broadcast / barrier through the C ABI."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tests._util import make_inputs  # noqa: E402
from torchx_b200.ddp import Communicator  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--device", type=int, required=True)
    ap.add_argument("--shm", required=True)
    ap.add_argument("--epoch", type=int, default=0)
    ap.add_argument("--n", type=int, default=100003)
    ap.add_argument("--out", required=True)
    ap.add_argument("--max-ctas", type=int, default=8)
    ap.add_argument("--op-count", type=int, default=0, help="the op counter every rank starts at")
    a = ap.parse_args()

    comm = Communicator.create(a.rank, a.world, a.device, a.shm, epoch=a.epoch, stage_mb=8, timeout_s=60)
    comm.set_timeout(30.0)
    comm.set_max_ctas(a.max_ctas)
    if a.op_count:
        comm.set_param("op_count", a.op_count)
    results = {}
    comm.set_param("pipe_chunk_bytes", 16 << 10)  # several pipeline chunks even at this message size
    for k, (algo, mode) in enumerate([("twoshot", "bf16"), ("oneshot", "bf16"), ("twoshot", "f32"), ("twoshot_pipe", "bf16")]):
        x = make_inputs(a.world, a.n, 10 + k, "special")[a.rank]
        t = torch.from_numpy(x).to(f"cuda:{a.device}")
        comm.allreduce_(t, wire=mode, algo=algo)
        results[f"ar{k}"] = t.cpu().numpy()
    x = make_inputs(a.world, a.n, 30, "special")[a.rank]
    t = torch.from_numpy(x).to(f"cuda:{a.device}")
    for _ in range(3):  # back to back on the same buffers: the sentinel reset / parity double-buffering / flow control
        t.copy_(torch.from_numpy(x))
        comm.allreduce_(t, wire="bf16", algo="twoshot_ll")
    results["ll"] = t.cpu().numpy()
    results["caps"] = np.array([comm.caps])
    if comm.has_multicast:  # NVLS through the multi-process multicast bring-up (fd passing, AddDevice / BindMem handshake)
        x = make_inputs(a.world, a.n, 20, "randn")[a.rank]
        t = torch.from_numpy(x).to(f"cuda:{a.device}")
        comm.allreduce_(t, wire="bf16", algo="nvls")
        results["nvls"] = t.cpu().numpy()
    b = torch.full((4097,), float(a.rank + 1), device=f"cuda:{a.device}")
    comm.broadcast_(b, root=a.world - 1)
    comm.barrier()
    torch.cuda.synchronize()
    comm.check()
    results["bcast"] = b.cpu().numpy()
    results["counted"] = np.array([comm.op_count - a.op_count == comm.launches])
    np.savez(a.out, **results)
    comm.close()
    print(f"rank {a.rank} ok", flush=True)


if __name__ == "__main__":
    main()
