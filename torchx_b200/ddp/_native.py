"""ctypes binding of libb200ddp.so (include/b200ddp.h).  No torch types cross this boundary: tensors are
passed as ``data_ptr()`` + element counts and streams as raw ``cudaStream_t`` values.

There is deliberately NO fallback: if the shared library is missing the import of the data plane raises,
so a GPU box can never silently run a CPU or library path in its place.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Optional

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(_PKG, "lib", "libb200ddp.so")
SRC_DIR = os.path.join(_PKG, "csrc")
SRC_PATH = os.path.join(SRC_DIR, "b200ddp.cu")  # the one translation unit; it includes the other files of csrc/
INCLUDE_DIR = os.path.join(os.path.dirname(_PKG), "include")

B2_ABI_VERSION = 3
B2_MAX_WORLD = 8

B2_OK = 0
B2_EINVAL = -1
B2_ECUDA = -2
B2_ESYS = -3
B2_ETIMEOUT = -4
B2_ENOPEER = -5
B2_ESTATE = -6
B2_ENOTSUP = -7

B2_F32_WIRE_BF16 = 0
B2_F32 = 1
B2_BF16 = 2
B2_F32_WIRE_F16 = 3
B2_F16 = 4

B2_ALGO_AUTO = 0
B2_ALGO_ONESHOT = 1
B2_ALGO_TWOSHOT = 2
B2_ALGO_TWOSHOT_PIPE = 3
B2_ALGO_NVLS = 4
B2_ALGO_TWOSHOT_LL = 5

B2_CAP_VMM = 1
B2_CAP_MULTICAST = 2

B2_DT_INT32 = 0
B2_DT_INT64 = 1
B2_DT_FLOAT32 = 2
B2_DT_BFLOAT16 = 3
B2_DT_FLOAT16 = 4

B2_OP_SUM = 0
B2_OP_AVG = 1
B2_OP_MIN = 2
B2_OP_MAX = 3

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-O3",
    "-lineinfo",
    "-std=c++17",
    "-Xcompiler",
    "-fPIC",
    "-shared",
]

B2_MAX_SEGMENTS = 128
B2_SEGMENT_ZEROS = 1  # a segment's src: its elements read as +0.0 (a parameter without a gradient this step)


class B2Segment(ctypes.Structure):
    """b2_segment_t: bucket elements [begin, end) live at device pointer src."""

    _fields_ = [("src", ctypes.c_void_p), ("begin", ctypes.c_uint64), ("end", ctypes.c_uint64)]


B2_P2P_MAX_OPS = 64


class B2P2pOp(ctypes.Structure):
    """b2_p2p_op_t: one send (is_send != 0) or receive of `bytes` bytes at device pointer ptr, to or from rank peer."""

    _fields_ = [("peer", ctypes.c_int), ("is_send", ctypes.c_int), ("ptr", ctypes.c_void_p), ("bytes", ctypes.c_size_t)]


B2_OPT_SGD = 1
B2_OPT_ADAM = 2
B2_OPT_ADAMW = 3
B2_OPT_MAX_GROUPS = 8
B2_OPT_MAX_RUNS = 128
B2_OPT_NO_GROUP = 255


class B2OptimGroup(ctypes.Structure):
    """b2_optim_group_t: one parameter group's hyper-parameters, as the optimizer's param_groups hold them."""

    _fields_ = [("lr", ctypes.c_double), ("weight_decay", ctypes.c_double), ("momentum", ctypes.c_double),
                ("dampening", ctypes.c_double), ("beta1", ctypes.c_double), ("beta2", ctypes.c_double),
                ("eps", ctypes.c_double), ("nesterov", ctypes.c_int), ("maximize", ctypes.c_int)]


class B2Optim(ctypes.Structure):
    """b2_optim_t: the optimizer step fused into b2_reduce_scatter_step."""

    _fields_ = [("kind", ctypes.c_int), ("n_groups", ctypes.c_int), ("n_runs", ctypes.c_int),
                ("param", ctypes.c_void_p), ("state0", ctypes.c_void_p), ("state1", ctypes.c_void_p),
                ("run_begin", ctypes.c_uint64 * (B2_OPT_MAX_RUNS + 1)), ("run_group", ctypes.c_uint8 * B2_OPT_MAX_RUNS),
                ("run_step", ctypes.c_float * B2_OPT_MAX_RUNS), ("run_index", ctypes.c_uint64 * B2_OPT_MAX_RUNS),
                ("run_scalar", ctypes.c_uint8 * B2_OPT_MAX_RUNS), ("group", B2OptimGroup * B2_OPT_MAX_GROUPS)]


_vp, _i, _sz, _u64, _f, _d = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_float, ctypes.c_double
_P = ctypes.POINTER

# name -> (restype, argtypes) of every symbol include/b200ddp.h declares (tests/test_abi.py checks the header and SYMBOLS agree)
SIGNATURES = {
    "b2_version": (_i, []),
    "b2_last_error": (ctypes.c_char_p, []),
    "b2_comm_create": (_i, [_P(_vp), _i, _i, _i, ctypes.c_char_p, _u64, _sz, _i]),
    "b2_comm_create_local": (_i, [_P(_vp), _i, _P(_i), _sz]),
    "b2_comm_destroy": (_i, [_vp]),
    "b2_comm_rank": (_i, [_vp]),
    "b2_comm_world": (_i, [_vp]),
    "b2_comm_device": (_i, [_vp]),
    "b2_comm_caps": (_i, [_vp]),
    "b2_comm_set_timeout_ms": (_i, [_vp, _i]),
    "b2_comm_set_max_ctas": (_i, [_vp, _i]),
    "b2_comm_set_param": (_i, [_vp, ctypes.c_char_p, ctypes.c_longlong]),
    "b2_comm_status": (_i, [_vp]),
    "b2_comm_op_count": (_u64, [_vp]),
    "b2_comm_launch_count": (_u64, [_vp]),
    "b2_comm_last_algo": (_i, [_vp]),
    "b2_auto_algo": (_i, [_i, _i, _sz, _i]),
    "b2_comm_trace": (_i, [_vp, _i, _P(_u64), _i]),
    "b2_allreduce": (_i, [_vp, _vp, _sz, _i, _f, _i, _vp]),
    "b2_allreduce_gather": (_i, [_vp, _vp, _sz, _P(B2Segment), _i, _i, _f, _i, _vp]),
    "b2_broadcast": (_i, [_vp, _vp, _sz, _i, _vp]),
    "b2_allreduce_op": (_i, [_vp, _vp, _sz, _i, _i, _vp]),
    "b2_allgather": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "b2_reduce_scatter": (_i, [_vp, _vp, _vp, _sz, _i, _i, _vp]),
    "b2_reduce": (_i, [_vp, _vp, _sz, _i, _i, _i, _vp]),
    "b2_reduce_scatter_gather": (_i, [_vp, _vp, _sz, _P(B2Segment), _i, _i, _f, _vp]),
    "b2_reduce_scatter_step": (_i, [_vp, _sz, _P(B2Segment), _i, _i, _f, _P(B2Optim), _vp]),
    "b2_reduce_scatter_step_bf16": (_i, [_vp, _sz, _P(B2Segment), _i, _f, _P(B2Optim), _vp, _vp]),
    "b2_alltoall": (_i, [_vp, _P(_vp), _P(_sz), _P(_vp), _P(_sz), _vp]),
    "b2_alltoall_max_bytes": (_sz, [_vp]),
    "b2_p2p": (_i, [_vp, _P(B2P2pOp), _i, _vp]),
    "b2_p2p_eager_bytes": (_sz, [_vp]),
    "b2_batchnorm_stats": (_i, [_vp, _vp, _vp, _f, _sz, _vp, _vp, _d, _d, _vp, _vp]),
    "b2_bn_forward_elemt": (_i, [_vp, _vp, _sz, _sz, _i, _vp, _vp, _vp, _vp, _d, _vp, _i, _vp]),
    "b2_bn_backward_elemt": (_i, [_vp, _vp, _vp, _sz, _sz, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "b2_bn_reduce_plan": (_i, [_sz, _sz, _P(_i), _P(_sz)]),
    "b2_bn_stats": (_i, [_vp, _sz, _sz, _i, _vp, _vp, _vp, _vp, _d, _vp, _sz, _i, _vp]),
    "b2_bn_backward_reduce": (_i, [_vp, _vp, _sz, _sz, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _i, _vp]),
    "b2_barrier": (_i, [_vp, _vp]),
    "b2_local_pass": (_i, [_vp, _sz, _i, _f, _i, _vp]),
}
SYMBOLS = list(SIGNATURES)


class B2Error(RuntimeError):
    def __init__(self, code: int, msg: str) -> None:
        super().__init__(f"libb200ddp error {code}: {msg}")
        self.code = code


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile torchx_b200/csrc/b200ddp.cu for sm_90a into torchx_b200/lib/ (in-tree, next to the package that
    loads it).  nvcc cross-compiles without a GPU."""
    os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
    hdr = os.path.join(INCLUDE_DIR, "b200ddp.h")
    # this file too: a library built with other NVCC_FLAGS (another architecture) is stale
    sources = [hdr, os.path.abspath(__file__)] + [os.path.join(SRC_DIR, f) for f in os.listdir(SRC_DIR) if f.endswith((".cu", ".cuh", ".h"))]
    newest = max(os.path.getmtime(f) for f in sources)
    if not force and os.path.exists(LIB_PATH) and os.path.getmtime(LIB_PATH) >= newest:
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc, *NVCC_FLAGS, SRC_PATH, "-o", LIB_PATH, "-lrt"]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.run(cmd, check=True)
    return LIB_PATH


_lib: Optional[ctypes.CDLL] = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: the CUDA data plane has not been built. Run "
            "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). There is no CPU fallback."
        )
    L = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype = restype
        fn.argtypes = argtypes
    if L.b2_version() != B2_ABI_VERSION:
        raise ImportError(f"libb200ddp ABI {L.b2_version()} != binding {B2_ABI_VERSION}; rebuild")
    _lib = L
    return L


def check(rc: int) -> None:
    if rc != B2_OK:
        raise B2Error(rc, lib().b2_last_error().decode("utf-8", "replace"))
