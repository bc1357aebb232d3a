"""Every kernel instance libb200ddp.so is built with, and the GPU test that launches it.

``LEDGER`` maps an instance's name, as ``tools/sass_report.demangle`` prints it (``k_oneshot<3, 5>``, ``k_pipe<0, 8, 1>``,
``k_barrier``), to where it runs:
  * ``tests/<file>.py``: a test of that file launches it;
  * ``tests/test_kernel_ledger_gpu.py::<test>``: that test launches it and checks, under ``torch.profiler``, that it did;
  * ``MULTICAST``: only a box with at least W GPUs bound into one NVSwitch multicast object can launch it.

The set is built from the constants of ``include/b200ddp.h`` and the instantiation rules of ``csrc/b200ddp.cu``:
``tests/test_kernel_ledger.py`` checks it against the built library, so a kernel instance added without a test that
launches it fails on a machine without a GPU.  Plain Python, no GPU and no package import."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = "tests/test_kernel_ledger_gpu.py"
MULTICAST = "multi-GPU with multicast"


def header_constants():
    """``#define B2_<NAME> <integer>`` of include/b200ddp.h -> {name: value}."""
    with open(os.path.join(ROOT, "include", "b200ddp.h")) as f:
        return {k: int(v) for k, v in re.findall(r"^#define\s+(B2_\w+)\s+(-?\d+)\b", f.read(), flags=re.M)}


H = header_constants()
MAX_WORLD = H["B2_MAX_WORLD"]
WORLDS = range(2, MAX_WORLD + 1)                          # the compile-time worlds of with_world
MODES = [H[k] for k in ("B2_F32_WIRE_BF16", "B2_F32", "B2_BF16", "B2_F32_WIRE_F16", "B2_F16")]  # with_mode
F16_MODES = {H["B2_F32_WIRE_F16"], H["B2_F16"]}
SUM_MODES = [H["B2_F32"], H["B2_BF16"], H["B2_F16"]]       # sum_mode_for: the modes of a float SUM / AVG (k_reduce)
STEP_MODES = [H["B2_F32_WIRE_BF16"], H["B2_F32"], H["B2_BF16"], H["B2_F32_WIRE_F16"]]  # k_reduce_scatter_step, k_local_step
INT_DTYPES = [H["B2_DT_INT32"], H["B2_DT_INT64"]]
FLOAT_DTYPES = [H["B2_DT_FLOAT32"], H["B2_DT_BFLOAT16"], H["B2_DT_FLOAT16"]]
# with_exact_op: integer SUM, and MIN / MAX on every dtype (float SUM / AVG run on the gradient kernels)
EXACT = ([(dt, H[op]) for dt in INT_DTYPES for op in ("B2_OP_SUM", "B2_OP_MIN", "B2_OP_MAX")]
         + [(dt, H[op]) for dt in FLOAT_DTYPES for op in ("B2_OP_MIN", "B2_OP_MAX")])
K_NVLS, K_P2P = 0, 1  # k_pipe's third argument (pl::kNvls, pl::kP2p)
NEW_WORLDS = (5, 6, 7)  # the worlds only test_kernel_ledger_gpu.py runs (and test_zero_segments_gpu.py, in modes 0-2)


def _ledger():
    led = {}

    def add(name, where):
        assert name not in led, name
        led[name] = where

    # one rank: the fused cast / scale pass (plain and TMA-staged), its optimizer twin, BatchNorm2d's four passes
    for m in MODES:
        f = "tests/test_fp16_gpu.py" if m in F16_MODES else "tests/test_allreduce_gpu.py"
        add(f"k_local_pass<{m}>", f)
        add(f"k_local_pass_tma<{m}>", f)
    for m in STEP_MODES:
        add(f"k_local_step<{m}>", "tests/test_zero_master_gpu.py" if m == H["B2_BF16"] else "tests/test_zero_overlap_gpu.py")
    for k in ("k_bn2d_norm<4>", "k_bn2d_bwd_elemt<2>", "k_bn2d_stats<4>", "k_bn2d_stats_merge", "k_bn2d_bwd_reduce<2>",
              "k_bn2d_bwd_reduce_merge"):
        add(k, f"{NEW}::test_batchnorm_column_tiles")
    # world a run-time value
    add("k_barrier", "tests/test_allreduce_gpu.py")
    add("k_broadcast", "tests/test_allreduce_gpu.py")
    add("k_allgather", "tests/test_exact_ops_gpu.py")
    add("k_alltoall", "tests/test_alltoall_gpu.py")
    add("k_p2p", "tests/test_p2p_gpu.py")
    add("k_bn_stats", "tests/test_syncbn_gpu.py")
    for dt, op in EXACT:
        add(f"k_reduce_exact<{dt}, {op}>", "tests/test_exact_ops_gpu.py")
        add(f"k_reduce_scatter_exact<{dt}, {op}>", "tests/test_reduce_scatter_gpu.py")
        add(f"k_reduce_exact_root<{dt}, {op}>", "tests/test_reduce_gpu.py")
    # one instance per (mode, world)
    for W in WORLDS:
        new = W in NEW_WORLDS
        for m in MODES:
            f16 = m in F16_MODES
            if new:
                where = f"{NEW}::test_allreduce" if f16 else "tests/test_zero_segments_gpu.py"
            else:
                where = "tests/test_fp16_gpu.py" if f16 else "tests/test_allreduce_gpu.py"
            for k in ("k_oneshot", "k_twoshot", "k_ll"):
                add(f"{k}<{m}, {W}>", where)
            add(f"k_pipe<{m}, {W}, {K_P2P}>", where)
            add(f"k_pipe<{m}, {W}, {K_NVLS}>", MULTICAST)
            rs_old = "tests/test_reduce_scatter_gpu.py" if m in SUM_MODES else "tests/test_zero_gpu.py"
            add(f"k_reduce_scatter<{m}, {W}>", f"{NEW}::test_reduce_scatter" if new else rs_old)
        for m in STEP_MODES:
            old = "tests/test_zero_master_gpu.py" if m == H["B2_BF16"] else "tests/test_zero_overlap_gpu.py"
            add(f"k_reduce_scatter_step<{m}, {W}>", f"{NEW}::test_fused_step" if new else old)
        for m in SUM_MODES:
            add(f"k_reduce<{m}, {W}>", f"{NEW}::test_reduce" if new else "tests/test_reduce_gpu.py")
    return led


LEDGER = _ledger()


def template_args(name):
    """``k_pipe<0, 5, 1>`` -> (0, 5, 1); ``k_barrier`` -> ()."""
    m = re.search(r"<([^>]*)>", name)
    return tuple(int(a) for a in m.group(1).split(",")) if m else ()


def assigned_to(test, **args):
    """The ledger entries ``tests/test_kernel_ledger_gpu.py::<test>`` launches; ``world=W`` / ``mode=M`` keep those whose
    template arguments are <M, W, ...>."""
    out = set()
    for name, where in LEDGER.items():
        if where != f"{NEW}::{test}":
            continue
        a = template_args(name)
        if "mode" in args and a[:1] != (args["mode"],):
            continue
        if "world" in args and a[1:2] != (args["world"],):
            continue
        out.add(name)
    return out
