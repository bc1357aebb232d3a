"""DDP communication hook backed by the fused H100 kernel: drop-in for
``torch.distributed.algorithms.ddp_comm_hooks.default_hooks.bf16_compress_hook`` (default_hooks.py:57-93) on a stock
``torch.nn.parallel.DistributedDataParallel`` - same signature ``hook(state, bucket) -> Future[Tensor]``
(torch/nn/parallel/distributed.py:1987-2067; DDP inspects the return annotation, so it must be the real type, not a
string), same result semantics (bucket averaged over ranks, values rounded to
bf16 and widened back to fp32), one launch instead of four and no NCCL on the data path.

    ddp = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local_rank])
    ddp.register_comm_hook(B200HookState(comm), b200_bf16_compress_hook)

``b200_fp16_compress_hook`` is the same for ``default_hooks.fp16_compress_hook`` (fp16 on the wire).  A bf16 or fp16
bucket (a ``.bfloat16()`` / ``.half()`` model) is reduced in its own format by every hook, as ``allreduce_hook`` would.
"""
from typing import Optional

import torch

from .comm import Communicator


class B200HookState:
    def __init__(self, comm: Optional[Communicator] = None, wire: str = "bf16", algo: str = "auto") -> None:
        if comm is None:  # one communicator per process: reuse the one init_pg("b200") created (each owns a multi-GiB arena)
            from torchx_b200 import distributed as _dist

            comm = _dist._COMM if _dist._COMM is not None else Communicator.from_env()
        self.comm = comm
        self.wire = wire
        self.algo = algo
        self.device = torch.device("cuda", self.comm.device)
        self.stream = torch.cuda.Stream(device=self.device)
        self.event = torch.cuda.Event()


def _run(state: B200HookState, bucket, wire: str) -> torch.futures.Future[torch.Tensor]:
    buf = bucket.buffer()
    cur = torch.cuda.current_stream(state.device)
    state.event.record(cur)  # the Reducer filled the bucket on the backward stream
    state.stream.wait_event(state.event)
    state.comm.allreduce_(buf, scale=1.0 / state.comm.world, wire=wire, algo=state.algo, stream=state.stream)
    fut: torch.futures.Future[torch.Tensor] = torch.futures.Future(devices=[state.device])
    with torch.cuda.stream(state.stream):
        fut.set_result(buf)  # the CUDA future captures an event on state.stream; fut.wait() orders consumers after it
    return fut


def b200_bf16_compress_hook(state: B200HookState, bucket) -> torch.futures.Future[torch.Tensor]:
    return _run(state, bucket, "bf16")


def b200_fp16_compress_hook(state: B200HookState, bucket) -> torch.futures.Future[torch.Tensor]:
    """Drop-in for ``default_hooks.fp16_compress_hook``: the bucket is cast to fp16, divided by W, summed and widened back
    (values rounded to fp16; an overflow arrives as inf on every rank, which is what GradScaler looks for)."""
    return _run(state, bucket, "f16")


def b200_allreduce_hook(state: B200HookState, bucket) -> torch.futures.Future[torch.Tensor]:
    """fp32-wire variant == default DDP semantics (pre-divide by W, SUM in fp32)."""
    return _run(state, bucket, "f32")
