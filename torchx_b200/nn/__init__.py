"""Layers that need the native communicator: ``SyncBatchNorm``."""
from .batchnorm import SyncBatchNorm  # noqa: F401
