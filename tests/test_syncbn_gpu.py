"""SyncBatchNorm's statistics exchange on the GPU: b2_batchnorm_stats bit for bit against torch.batch_norm_gather_stats_with_
counts on the rows torch's own mask keeps, W = 1 .. 8 ranks sharing one device, with guard bands, misaligned views and
interleaved with the other collectives; torchx_b200.nn.SyncBatchNorm in worker processes against torch's code path, and
against torch.nn.SyncBatchNorm itself over gloo (every rank on one GPU) and over NCCL (one GPU per rank, skipped on a box with
fewer than two); and the module under the mini-DDP."""
import os
import socket
import subprocess
import sys
import uuid

import numpy as np
import pytest
import torch

from tests._util import GUARD, World, assert_bits_equal, assert_guards_intact

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POISON = 1e30


def count_patterns(world):
    pats = [[64.0] * world, [float(3 + 17 * r) for r in range(world)]]
    if world > 1:
        pats.append([0.0 if r % 2 else float(5 + r) for r in range(world)])  # empty ranks in between
        pats.append([0.0] * (world - 1) + [1.0])
    else:
        pats.append([1.0])
    pats.append([0.0] * world)  # nobody has a sample: torch's masked path on no rows
    return pats


def padded(vals, off):
    h = np.concatenate([np.full(off, POISON, np.float32), vals.astype(np.float32), np.full(GUARD, POISON, np.float32)])
    return h, torch.from_numpy(h.copy()).cuda()


def check_stats(w, C, counts, running, momentum, eps, off, seed, with_counts=True):
    """running = (running_mean given, running_var given): either may be absent on its own."""
    W = len(w.comms)
    rng = np.random.default_rng(seed)
    means = (rng.standard_normal((W, C)) * 3).astype(np.float32)
    invs = rng.uniform(0.2, 5.0, (W, C)).astype(np.float32)
    rms = rng.standard_normal((W, C)).astype(np.float32)
    rvs = rng.uniform(0.5, 2.0, (W, C)).astype(np.float32)
    bufs = []
    for r in range(W):
        b = {k: padded(v, off) for k, v in (("mean", means[r]), ("invstd", invs[r]), ("rm", rms[r]), ("rv", rvs[r]),
                                            ("counts", np.zeros(W, np.float32)))}
        bufs.append(b)
    view = lambda b, k, n: b[k][1][off:off + n]  # noqa: E731

    def launch(r, c, s):
        b = bufs[r]
        c.batchnorm_stats_(view(b, "mean", C), view(b, "invstd", C), counts[r], view(b, "rm", C) if running[0] else None,
                           view(b, "rv", C) if running[1] else None, momentum=momentum, eps=eps,
                           counts_out=view(b, "counts", W) if with_counts else None, stream=s)

    w.run(launch)
    what = f"W={W} C={C} counts={counts} running={running} counts_out={with_counts} momentum={momentum} eps={eps} off={off}"
    mask = torch.tensor(counts) >= 1
    dummy = torch.zeros(2, C, device="cuda")  # the `input` argument only selects ATen's <float, float, int32_t> instance
    for r in range(W):
        rm, rv = torch.from_numpy(rms[r]).cuda(), torch.from_numpy(rvs[r]).cuda()
        wm, wi = torch.batch_norm_gather_stats_with_counts(
            dummy, torch.from_numpy(means).cuda()[mask.cuda()], torch.from_numpy(invs).cuda()[mask.cuda()],
            rm if running[0] else None, rv if running[1] else None, momentum, eps,
            torch.tensor(counts, device="cuda")[mask.cuda()])
        b = bufs[r]
        for k, want, n in (("mean", wm, C), ("invstd", wi, C), ("rm", rm if running[0] else None, C),
                           ("rv", rv if running[1] else None, C), ("counts", torch.tensor(counts) if with_counts else None, W)):
            got = b[k][1].cpu().numpy()
            before = b[k][0]
            assert_guards_intact(got, before, off, off + n, f"{what} rank={r} {k}")
            if want is not None:
                assert_bits_equal(got[off:off + n], want.cpu().numpy().astype(np.float32), f"{what} rank={r} {k}")
            else:
                assert got.view(np.uint32).tolist() == before.view(np.uint32).tolist(), f"{what} rank={r} {k} written"


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_kernel_matches_aten_gather_stats(world):
    w = World([0] * world)
    settings = [(0.1, 1e-5), (0.01, 1e-3), (1.0, 0.0), (0.3, 0.5)]
    try:
        k = 0
        for C in (1, 3, 64, 2048, 4099):
            for counts in count_patterns(world):
                momentum, eps = settings[k % len(settings)]
                running = ((True, True), (False, False), (True, False), (False, True))[k % 4]
                check_stats(w, C, counts, running=running, momentum=momentum, eps=eps, off=(k // 2) % 3, seed=k,
                            with_counts=k % 3 != 2)
                k += 1
    finally:
        w.close()


def test_row_larger_than_a_stage_region_is_refused():
    from torchx_b200.ddp import _native as N

    w = World([0] * 2, stage_mb=1)
    try:
        t = torch.zeros(200_000, device="cuda")
        with pytest.raises(N.B2Error, match="need a .*-byte row, a stage region holds"):
            w.comms[0].batchnorm_stats_(t, t.clone(), 3.0, momentum=0.1, eps=1e-5)
        assert w.comms[0].launches == 0
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_interleaved_with_the_other_collectives(world):
    """Rounds of bucket allreduce_, allreduce_op_, allgather_, broadcast_ and batchnorm_stats_ back to back without a host
    sync: five collectives a round, so the statistics exchange runs on both stage parities."""
    from tests import _exact_oracle as X
    import oracle

    w = World([0] * world)
    rounds, n, C = 6, 1000, 70
    try:
        plan = []
        for k in range(rounds):
            rng = np.random.default_rng(k)
            p = dict(b=[rng.standard_normal(n).astype(np.float32) for _ in range(world)],
                     i=[rng.integers(-100, 100, n).astype(np.int64) for _ in range(world)],
                     g=[rng.integers(0, 1000, 37).astype(np.int32) for _ in range(world)],
                     bc=[np.full(n + 3, (r + 10 * k) % 256, np.uint8) for r in range(world)],
                     m=(rng.standard_normal((world, C))).astype(np.float32), s=rng.uniform(0.5, 2, (world, C)).astype(np.float32),
                     cnt=[float(rng.integers(0, 4) * (r + 1)) for r in range(world)], root=k % world)
            p["tb"] = [torch.from_numpy(x.copy()).cuda() for x in p["b"]]
            p["ti"] = [torch.from_numpy(x.copy()).cuda() for x in p["i"]]
            p["tg"] = [torch.from_numpy(x.copy()).cuda() for x in p["g"]]
            p["tgo"] = [torch.empty(world * 37, dtype=torch.int32, device="cuda") for _ in range(world)]
            p["tc"] = [torch.from_numpy(x.copy()).cuda() for x in p["bc"]]
            p["tm"] = [torch.from_numpy(p["m"][r].copy()).cuda() for r in range(world)]
            p["ts"] = [torch.from_numpy(p["s"][r].copy()).cuda() for r in range(world)]
            plan.append(p)
        torch.cuda.synchronize()

        def ops(r, c, s, p):
            return [lambda: c.allreduce_(p["tb"][r], wire="bf16", stream=s),
                    lambda: c.allreduce_op_(p["ti"][r], "max", stream=s),
                    lambda: c.allgather_(p["tgo"][r], p["tg"][r], stream=s),
                    lambda: c.broadcast_(p["tc"][r], root=p["root"], stream=s),
                    lambda: c.batchnorm_stats_(p["tm"][r], p["ts"][r], p["cnt"][r], momentum=0.1, eps=1e-5, stream=s)]

        # load every kernel first, one synchronised op at a time (see test_exact_ops_gpu.py: lazy module loading)
        scratch = {k: ([t.clone() for t in v] if k.startswith("t") else v) for k, v in plan[0].items()}
        for o in range(5):
            w.run(lambda r, c, s: ops(r, c, s, scratch)[o]())

        def issue(r, c, s):
            for p in plan:
                for op in ops(r, c, s, p):
                    op()

        w.run(issue)
        for k, p in enumerate(plan):
            mask = torch.tensor(p["cnt"]) >= 1
            wm, wi = torch.batch_norm_gather_stats_with_counts(
                torch.zeros(2, C, device="cuda"), torch.from_numpy(p["m"]).cuda()[mask.cuda()],
                torch.from_numpy(p["s"]).cuda()[mask.cuda()], None, None, 0.1, 1e-5,
                torch.tensor(p["cnt"], device="cuda")[mask.cuda()])
            wb = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, p["b"], 1.0 / world)
            wi64 = X.reduce("int64", "max", p["i"])
            for r in range(world):
                assert_bits_equal(p["tb"][r].cpu().numpy(), wb, f"round {k} bucket rank {r}")
                assert np.array_equal(p["ti"][r].cpu().numpy(), wi64.view(np.int64)), f"round {k} max rank {r}"
                assert np.array_equal(p["tgo"][r].cpu().numpy().view(np.uint8), X.allgather(p["g"])), f"round {k} gather rank {r}"
                assert np.array_equal(p["tc"][r].cpu().numpy(), p["bc"][p["root"]]), f"round {k} broadcast rank {r}"
                assert_bits_equal(p["tm"][r].cpu().numpy(), wm.cpu().numpy(), f"round {k} bn mean rank {r}")
                assert_bits_equal(p["ts"][r].cpu().numpy(), wi.cpu().numpy(), f"round {k} bn invstd rank {r}")
    finally:
        w.close()


def run_workers(tmp_path, world, mode, devices=None, extra=()):
    shm = f"/b2_sbn_{uuid.uuid4().hex[:12]}"
    devices = devices or [0] * world
    procs = []
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "syncbn_worker.py"), "--rank", str(r), "--world", str(world),
               "--device", str(devices[r]), "--shm", shm, "--mode", mode, "--out", str(tmp_path / f"{mode}{r}.npz"), *extra]
        procs.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            o, _ = p.communicate(timeout=600)
            outs.append(o)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, p in enumerate(procs):
        assert p.returncode == 0, f"rank {r} failed:\n{outs[r]}"
    return [dict(np.load(tmp_path / f"{mode}{r}.npz")) for r in range(world)]


@pytest.mark.parametrize("world", [2, 4])
def test_module_matches_torchs_code_path(tmp_path, world):
    """Forward output, running statistics and grad_input of every rank bit-equal to torch's SyncBatchNorm code path run in
    one process (exact concatenation for the all_gather, rank-order fp32 sum for the allreduce), in fp32 and bf16 under
    autocast, NCHW, channels_last and NC, unequal batch sizes and empty ranks; and no host sync (sync debug mode "error")."""
    res = run_workers(tmp_path, world, "module")
    for r, got in enumerate(res):
        assert int(got["nosync.ok"]) == 1
        keys = sorted(k[:-4] for k in got if k.endswith(".got"))
        assert len(keys) == 7 * 4
        for k in keys:
            g, wv = got[k + ".got"], got[k + ".want"]
            assert g.shape == wv.shape, (r, k)
            assert g.tobytes() == wv.tobytes(), f"rank {r} {k}: {np.count_nonzero(g != wv)} of {g.size} differ"


@pytest.mark.parametrize("world", [2, 4])
def test_under_the_mini_ddp(tmp_path, world):
    """Buckets fire while SyncBatchNorm's backward collectives are still being issued; parameters and running statistics
    end identical on every rank and equal to the same training without overlap."""
    res = run_workers(tmp_path, world, "ddp")
    keys = [k[4:] for k in res[0] if k.startswith("ddp.")]
    assert any("running_mean" in k for k in keys)
    for r in range(world):
        for k in keys:
            assert res[r]["ddp." + k].tobytes() == res[0]["ddp." + k].tobytes(), f"rank {r} {k} differs from rank 0"
            assert res[r]["ddp." + k].tobytes() == res[r]["ref." + k].tobytes(), f"rank {r} {k} differs from the reference run"


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def check_against_torch(res, world):
    """torch.nn.SyncBatchNorm's own forward (outputs, running statistics, num_batches_tracked over several training steps and
    an eval step) against this package's on the fabric, bit for bit at every W: the gather is exact and the merge is ATen's.
    Gradients: weight and bias are local, equal at every W; grad_input goes through the backend's sum of (sum_dy,
    sum_dy_xmu), bit-equal at W = 2 (one add) only.  The trained conv net (mini-DDP against dist.all_reduce + 1/W): W = 2."""
    for r, got in enumerate(res):
        keys = [k[len("torch."):] for k in got if k.startswith("torch.")]
        assert keys and all("fabric." + k in got for k in keys), r
        assert any(k.endswith(".out") for k in keys) and any(".num_batches_tracked" in k for k in keys)
        for k in keys:
            if (".grad_input" in k or k.startswith("train.")) and world != 2:
                continue
            t, f = got["torch." + k], got["fabric." + k]
            assert t.shape == f.shape and t.tobytes() == f.tobytes(), f"rank {r} {k}: {np.count_nonzero(t != f)} of {t.size} differ"


@pytest.mark.parametrize("world", [2, 4])
def test_module_matches_torch_syncbatchnorm_over_gloo_one_gpu(tmp_path, world):
    """torch's real SyncBatchNorm (momentum None, no running statistics, no affine, an empty rank, bf16 autocast, eval) over
    a gloo group with every rank on cuda:0, against this package's under init_pg("b200")."""
    res = run_workers(tmp_path, world, "torch", extra=("--backend", "gloo", "--port", str(free_port())))
    check_against_torch(res, world)


@pytest.mark.parametrize("world", ["2", "all"])
def test_module_matches_torch_syncbatchnorm_over_nccl(tmp_path, world, cuda_count):
    """The same with one GPU per rank: torch's SyncBatchNorm over NCCL at W = 2 and at every GPU of the box."""
    if cuda_count < 2:
        pytest.skip("needs 2 GPUs")
    W = 2 if world == "2" else cuda_count
    res = run_workers(tmp_path, W, "torch", devices=list(range(W)), extra=("--backend", "nccl", "--port", str(free_port())))
    check_against_torch(res, W)
