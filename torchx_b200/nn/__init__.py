"""Layers with native kernels: ``SyncBatchNorm`` on the native communicator, ``BatchNorm2d`` on channels-last bf16 / fp16."""
from .batchnorm import SyncBatchNorm  # noqa: F401
from .bn2d import BatchNorm2d, convert_batchnorm, native_eligible  # noqa: F401
