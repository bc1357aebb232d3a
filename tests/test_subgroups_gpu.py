"""Process subgroups on the GPU: W = 4 and W = 8 processes sharing one H100 under init_pg("b200"), groups made with
torchx_b200.distributed.new_group / new_subgroups_by_enumeration (tests/workers/subgroups_worker.py).  Every helper's
result on every group against the oracles over the members' inputs in group-rank order, p2p by global rank, the op
counters of the world and of each group, mini-DDP + ZeRO-1 and SyncBatchNorm in groups of 2 bit-equal to the same run as a
W = 2 world (with a world all_reduce issued from a gradient hook mid-backward), and no shm object left behind.  The
processes are time-sliced on one device, so nothing here measures NVLink."""
import glob
import os
import subprocess
import sys
import uuid

import numpy as np
import pytest
import torch

from tests import _exact_oracle as X
from tests.test_exact_ops_gpu import assert_float_sum_equal, float_sum_oracle

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "workers"))
import subgroups_worker as SW  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_workers(tmp_path, world, case, devices=None):
    devices = devices or [0] * world
    shm = f"/b2_sg_{uuid.uuid4().hex[:12]}"
    procs = []
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "subgroups_worker.py"), "--rank", str(r), "--world",
               str(world), "--device", str(devices[r]), "--shm", shm, "--case", case, "--out", str(tmp_path / f"{case}{r}.npz")]
        procs.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            o, _ = p.communicate(timeout=900)
            outs.append(o)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, p in enumerate(procs):
        assert p.returncode == 0, f"rank {r} failed:\n{outs[r]}"
    assert glob.glob(f"/dev/shm{shm}*") == [], "a control block outlived the run"
    return [dict(np.load(tmp_path / f"{case}{r}.npz")) for r in range(world)]


def f32(rank, seed, n=SW.N):
    return SW.bits(SW.data(rank, seed, n=n))


def check_group(res, i, members, world):
    G, seed, tag = len(members), 7 + i, f"g{i}"
    ar = float_sum_oracle("float32", [f32(m, seed) for m in members], 1.0) if G > 1 else f32(members[0], seed)
    mx = X.reduce("int64", "max", [SW.data(m, seed + 1, torch.int64).numpy() for m in members])
    rs = float_sum_oracle("float32", [f32(m, seed + 2, G * 64) for m in members], 1.0) if G > 1 else f32(members[0], seed + 2, 64)
    red = float_sum_oracle("float32", [f32(m, seed + 3) for m in members], 1.0) if G > 1 else f32(members[0], seed + 3)
    for gr, m in enumerate(members):
        g = res[m]
        what = f"group {members} rank {m}"
        assert_float_sum_equal("float32", g[f"{tag}.allreduce"], ar, what)
        X.assert_exact_equal("int64", g[f"{tag}.allreduce_max"], mx, what)
        assert np.array_equal(g[f"{tag}.world_between"].view(np.float32), np.full(5, float(sum(range(world))), np.float32))
        assert g[f"{tag}.allgather"].tolist() == [k + 100 * mm for mm in members for k in range(7)], what
        assert_float_sum_equal("float32", g[f"{tag}.reduce_scatter"], rs[gr * 64:(gr + 1) * 64], what)
        assert g[f"{tag}.broadcast"].view(np.float32).tolist() == [float(members[-1])] * 9, what
        assert g[f"{tag}.broadcast_group_src"].view(np.float32).tolist() == [float(members[0])] * 9, what
        if gr == 0:
            assert_float_sum_equal("float32", g[f"{tag}.reduce"], red, what)
            assert g[f"{tag}.gather"].view(np.float32).tolist() == [float(mm) for mm in members for _ in range(4)], what
        assert g[f"{tag}.alltoall"].tolist() == [1000 * mm + 3 * gr + k for mm in members for k in range(3)], what
        if G > 1:
            prv = members[(gr - 1) % G]
            assert g[f"{tag}.ring"].view(np.float32).tolist() == [float(prv)] * 11, what
            assert g[f"{tag}.sendrecv"].view(np.float32).tolist() == [float(prv)] * 11, what
            assert int(g[f"{tag}.sendrecv_src"][0]) == prv, what  # recv returns the global rank
        assert g[f"{tag}.scatter"].view(np.float32).tolist() == [float(10 * gr)] * 4, what
        assert g[f"{tag}.objects"].tolist() == members, what


@pytest.mark.parametrize("world,case", [(4, "pairs"), (4, "strided"), (4, "three"), (4, "single"), (4, "twice"),
                                        (8, "split2x4"), (8, "split4x2")])
def test_group_collectives_match_the_oracles(tmp_path, world, case):
    res = run_workers(tmp_path, world, case)
    groups = SW.CASES[case]
    for i, members in enumerate(groups):
        check_group(res, i, members, world)
    # the world counter moved by the world's ops alone: as many small all_reduces as the busiest rank's groups
    most = max(sum(r in g for g in groups) for r in range(world))
    for r in range(world):
        w0, w1 = res[r]["world.op_count"]
        assert w1 - w0 == most, (r, w0, w1)
    # each group's counter by its own collectives: the same sequence on every group of more than one rank, none on one
    deltas = {(i, m): int(np.diff(res[m][f"g{i}.op_count"])[0]) for i, g in enumerate(groups) for m in g}
    multi = {d for (i, m), d in deltas.items() if len(groups[i]) > 1}
    assert len(multi) <= 1 and all(d > 0 for d in multi), deltas
    assert all(d == 0 for (i, m), d in deltas.items() if len(groups[i]) == 1), deltas


def test_ddp_zero_and_syncbn_in_groups_of_two_equal_a_world_of_two(tmp_path):
    ref = run_workers(tmp_path, 2, "world2")
    res = run_workers(tmp_path, 4, "train")
    for r in range(4):
        g = r % 2
        for k in ("train.params.0", "train.params.1", "train.bn.y", "train.bn.dx", "train.bn.running"):
            assert np.array_equal(res[r][k], ref[g][k]), (r, k)
        for ov in (0, 1):  # the world all_reduce issued from the gradient hook, once per backward
            assert int(res[r][f"train.hooked.{ov}"][0]) == 3
            # starts at the global rank, summed over the 4 ranks once per backward: 6, 24, 96
            assert res[r][f"train.probe.{ov}"].view(np.float32).tolist() == [96.0] * 1000, (r, ov)


@pytest.mark.skipif(torch.cuda.device_count() < 4, reason="needs 4 GPUs")
def test_groups_across_devices(tmp_path):
    res = run_workers(tmp_path, 4, "pairs", devices=[0, 1, 2, 3])
    for i, members in enumerate(SW.CASES["pairs"]):
        check_group(res, i, members, 4)
