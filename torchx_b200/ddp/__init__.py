"""Worker-side data plane: communicator, DDP wrapper and comm hooks on libb200ddp.so."""
from .comm import Communicator, local_pass_, mode_for  # noqa: F401
from .ddp import DistributedDataParallel  # noqa: F401
from .hooks import B200HookState, b200_allreduce_hook, b200_bf16_compress_hook, b200_fp16_compress_hook  # noqa: F401
from .zero import ZeroRedundancyOptimizer  # noqa: F401
