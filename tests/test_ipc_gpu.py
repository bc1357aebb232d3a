"""The multi-process path: one process per rank, rendezvous through the shm control block, peer arenas
exchanged as VMM file descriptors (+ one NVSwitch multicast object) or, failing that, mapped with CUDA IPC.  On a 1-GPU box all ranks share cuda:0 (IPC between processes on one device; the
kernels time-slice, so this is a functional check only); with >= 2 GPUs each rank gets its own device."""
import os
import subprocess
import sys
import uuid

import numpy as np
import pytest

import oracle
from tests._util import assert_bits_equal, assert_nvls_result, make_inputs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_world(world, devices, tmp_path, n=100003, op_count=0):
    shm = f"/b2_test_{uuid.uuid4().hex[:12]}"
    procs = []
    for r in range(world):
        out = tmp_path / f"r{r}.npz"
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "ipc_worker.py"), "--rank", str(r), "--world",
               str(world), "--device", str(devices[r]), "--shm", shm, "--n", str(n), "--out", str(out), "--op-count", str(op_count)]
        procs.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            o, _ = p.communicate(timeout=240)
            outs.append(o)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, p in enumerate(procs):
        assert p.returncode == 0, f"rank {r} failed:\n{outs[r]}"
    modes = [oracle.B2O_F32_WIRE_BF16, oracle.B2O_F32_WIRE_BF16, oracle.B2O_F32, oracle.B2O_F32_WIRE_BF16]
    for r in range(world):
        got = np.load(tmp_path / f"r{r}.npz")
        for k, mode in enumerate(modes):
            xs = make_inputs(world, n, 10 + k, "special")
            assert_bits_equal(got[f"ar{k}"], oracle.allreduce(mode, xs, 1.0 / world), f"rank {r} op {k}")
        assert np.all(got["bcast"] == float(world)), r
        assert got["counted"].all(), f"rank {r}: the op counter did not advance by one per collective from {op_count}"
        assert_bits_equal(got["ll"], oracle.allreduce(oracle.B2O_F32_WIRE_BF16, make_inputs(world, n, 30, "special"), 1.0 / world), f"rank {r} LL two-shot")
        if "nvls" in got.files:  # the box exposes NVSwitch multicast: the worker also ran the NVLS algorithm
            assert_nvls_result(got["nvls"], make_inputs(world, n, 20, "randn"), 1.0 / world, oracle.B2O_F32_WIRE_BF16, f"nvls rank {r}")
    return int(np.load(tmp_path / "r0.npz")["caps"][0])


def test_two_processes_share_one_device(tmp_path):
    _run_world(2, [0, 0], tmp_path, n=20011)


def test_two_processes_share_one_device_from_op_count_2_29(tmp_path):
    """Both ranks start their counter at 2^29, where a 32-bit flag compare would take a never-written slot for a current
    one (tests/test_op_count_gpu.py)."""
    _run_world(2, [0, 0], tmp_path, n=20011, op_count=1 << 29)


def test_two_processes_share_one_device_cuda_ipc_backend(tmp_path, monkeypatch):
    """B2_VMM=0: the cudaMalloc + CUDA IPC arena (the fallback when file descriptors cannot be passed)."""
    monkeypatch.setenv("B2_VMM", "0")
    assert _run_world(2, [0, 0], tmp_path, n=20011) == 0


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu(world, tmp_path, cuda_count):
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    _run_world(world, list(range(world)), tmp_path)
