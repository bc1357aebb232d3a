"""The kernel instances no other one-device test launches, against their oracles: every multi-rank kernel at W = 5, 6, 7
(where vecs_per_trip drops to one vec per trip, k_ll's fp32-wire polling groups end ragged, a stage region is no power of
two and small messages leave ranks with empty slices), and BatchNorm2d's elementwise passes over more than one column
tile (C > 2048).  The checkers are the parity files' own; each test records its launches with torch.profiler (in a child
process) and asserts that every instance tests/_kernel_ledger.py gives it ran, so a dispatch that routed a call elsewhere
fails here too."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import _kernel_ledger as K
from tests import test_allreduce_gpu as AR
from tests import test_alltoall_gpu as AA
from tests import test_exact_ops_gpu as EX
from tests import test_fp16_gpu as FP16
from tests import test_gather_gpu as GG
from tests import test_native_bn_gpu as BN
from tests import test_reduce_gpu as RD
from tests import test_reduce_scatter_gpu as RS
from tests import test_syncbn_gpu as SB
from tests import test_zero_gpu as ZG
from tests import test_zero_master_gpu as ZM
from tests import test_zero_overlap_gpu as ZO
from tests._util import MODES, World
from torchx_b200.ddp import _native as N

pytestmark = pytest.mark.gpu

WORLDS = list(K.NEW_WORLDS)
ALGOS = ("oneshot", "twoshot", "twoshot_pipe", "twoshot_ll", "auto")
ALL_MODES = list(MODES) + list(FP16.MODES)  # f32_wire_bf16, f32, bf16 (oracle.allreduce); f32_wire_f16, f16 (_oracle_f16)
KINDS = ("randn", "special", "nanbits", "onehot")
F16_KIND = {"nanbits": "f16bits", "onehot": "big"}  # the fp16 checker's kinds for the same edges: 0xFFFF words, overflow
KERNEL = re.compile(r"\bk_\w+(?:<[^>]*>)?")
_CHILD = "B2_LEDGER_TEST_CHILD"  # set in the child process of _ran_in_child: the test it runs


def _kernels(sweep):
    """Runs sweep() under torch.profiler and returns the names of the library's kernels it launched, as the ledger spells them."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        sweep()
        torch.cuda.synchronize()
    return {m.group(0) for e in prof.events() for m in KERNEL.finditer(e.name)}


def _profiler_keeps_ranks_concurrent():
    """The sweeps profile W spinning kernels that must all be resident at once.  Kineto records with CUPTI's
    concurrent-kernel activity, which leaves kernels concurrent; a profiler that serialised them would make the ranks of a
    collective unable to meet.  One W = 2 call with a 2 s timeout says so before any sweep."""
    w = World([0, 0], timeout_s=2.0)
    try:
        x = [torch.ones(4096, device="cuda:0") for _ in range(2)]
        ran = _kernels(lambda: w.run(lambda r, c, s: c.allreduce_(x[r], algo="twoshot", stream=s)))
        assert "k_twoshot<0, 2>" in ran, ran
        assert all(torch.equal(t, torch.ones_like(t)) for t in x)
    finally:
        w.close()


def _ran_in_child(test, args, sweep, want, what):
    """sweep() under torch.profiler, asserting that every instance of `want` ran - in a child process that runs
    `test(**args)` again.  Kineto keeps process-wide state: after the long sweeps here, short profiler sessions later in the
    same process (tests/test_native_bn_reduce_gpu.py's) come back without their GPU records.  The child keeps the pytest
    process free of any profiler session."""
    if os.environ.get(_CHILD) == test:
        _profiler_keeps_ranks_concurrent()
        try:
            _assert_ran(_kernels(sweep), want, what)
        finally:
            for v in ZG._WORLDS.values():
                v.close()
            ZG._WORLDS.clear()
        return
    code = f"from tests import test_kernel_ledger_gpu as T; T.{test}(**{args!r})"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    p = subprocess.run(cmd, cwd=K.ROOT, env=dict(os.environ, **{_CHILD: test}), capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0, f"{test}({args}) failed in its child process:\n{p.stdout[-4000:]}\n{p.stderr[-12000:]}"


def _assert_ran(launched, want, what):
    missing = sorted(set(want) - launched)
    assert not missing, f"{what}: {len(missing)} instances never launched: {missing}"


def _flat(w, n, mode, algo, kind, seed, offset=0):
    """One allreduce_ of n elements on every rank against the mode's oracle, guard bands included."""
    if mode in FP16.MODES:
        FP16._check_allreduce(w, n, mode, algo, F16_KIND.get(kind, kind), seed, offset)
    else:
        AR._check_allreduce(w, n, mode, algo, kind, seed, offset)
    ran = {c.last_algo for c in w.comms}
    assert len(ran) == 1 and (algo == "auto" or ran == {algo}), (n, mode, algo, ran)


def _sizes(W, k=37):
    """V < W (n = 1, 9, 8 (W - 1)); slice boundaries (8 W k - 7, 8 W k, 8 W k + 1: Ls = k vecs); a grid that strides
    several times."""
    return [1, 9, 8 * (W - 1), 8 * W * k - 7, 8 * W * k, 8 * W * k + 1, (1 << 18) + 5]


def _gather(w, n, mode, algo, seed):
    """The segment-table path: the gathered bucket against the oracle, sources and guards unchanged."""
    W = len(w.comms)
    if mode in FP16.MODES:
        cuts = sorted({0, 1, 8 * W - 1, 8 * W * 37 + 1, n})
        FP16._gather_case(w, mode, algo, cuts, (1, 0, 7, 3), seed)
    else:
        GG._case(w, n, mode, algo, GG.LAYOUTS[seed % len(GG.LAYOUTS)], GG.PLACEMENTS[seed % 4], GG.KINDS[seed % 3], seed,
                 out_off=seed % 2)


@pytest.mark.parametrize("world", WORLDS)
def test_allreduce(world):
    """Flat and gathered allreduce, modes 0-4 x every P2P algorithm and AUTO; the pipelined kernel with 1 KiB chunks (K > 1,
    ragged cells) and with one chunk; then stage_mb=1, so that each message takes several launches (counted)."""
    W = world

    def sweep():
        w = World([0] * W)
        try:
            for m, mode in enumerate(ALL_MODES):
                for a, algo in enumerate(ALGOS):
                    for c in w.comms:
                        c.set_param("pipe_chunk_bytes", 1 << 10)
                    for i, n in enumerate(_sizes(W)):
                        _flat(w, n, mode, algo, KINDS[(i + m + a) % 4], seed=100 * m + 10 * a + i)
                    _flat(w, 4099, mode, algo, "randn", seed=7, offset=1)  # base misaligned by one element
                    _gather(w, 8 * W * 37 + 1, mode, algo, seed=m + a)
                    _gather(w, 70001, mode, algo, seed=m + a + 1)
                    if algo == "twoshot_pipe":  # one chunk: K = 1
                        for c in w.comms:
                            c.set_param("pipe_chunk_bytes", 0)
                        _flat(w, 8 * W * 37 + 1, mode, algo, "special", seed=9)
                        _flat(w, (1 << 18) + 5, mode, algo, "nanbits", seed=10)
        finally:
            w.close()
        w = World([0] * W, stage_mb=1)
        try:
            for c in w.comms:
                c.set_param("pipe_chunk_bytes", 32 << 10)
            n = (1 << 19) + 13
            for m, mode in enumerate(ALL_MODES):
                for algo in ALGOS[:4]:
                    before = w.comms[0].launches
                    _flat(w, n, mode, algo, KINDS[m % 4], seed=20 + m)
                    want = len(GG._launches(n, W, mode, algo, 1))
                    assert w.comms[0].launches - before == want >= 2, (mode, algo, w.comms[0].launches - before, want)
                before = w.comms[0].launches
                _flat(w, n, mode, "auto", "special", seed=30 + m)
                assert w.comms[0].launches - before >= 2, mode
        finally:
            w.close()

    _ran_in_child("test_allreduce", dict(world=W), sweep, K.assigned_to("test_allreduce", world=W), f"W={W}")


@pytest.mark.parametrize("world", WORLDS)
def test_reduce_scatter(world):
    """reduce_scatter_ for every dtype and op (in place, misaligned, chunked with the launch count checked), each block
    against the oracles and allreduce_op_; reduce_scatter_gather_ in modes 0-4 against the oracle's block and
    allreduce_gather_ on the same communicator."""
    W = world

    def sweep():
        w = World([0] * W)
        try:
            for dtype, ops in EX.OPS.items():
                for op in ops:
                    for i, n in enumerate((1, 9, 4095, (1 << 17) + 3)):
                        RS.check_rs(w, dtype, op, n, seed=i)
                    RS.check_rs(w, dtype, op, 4095, seed=50, in_off=1, out_off=3)
                    RS.check_rs(w, dtype, op, 4095, seed=52, in_place=True)
                    RS.check_rs(w, dtype, op, 4093, seed=53, in_off=1, in_place=True)
        finally:
            w.close()
        w = World([0] * W, stage_mb=1)
        slice_cap = ((1 << 20) // (W + 1)) & ~255
        n = 3 * (slice_cap // 2) + 5
        try:
            for dtype, ops in EX.OPS.items():
                for op in ops[:2]:
                    per_elem = {"float32": 4, "int32": 4, "int64": 8}.get(dtype, 2)
                    before = w.comms[0].launches
                    RS.check_rs(w, dtype, op, n, seed=7, in_off=1, out_off=3, against_allreduce=False)
                    assert w.comms[0].launches - before == -(-n // (slice_cap // per_elem)) >= 3, (dtype, op)
        finally:
            w.close()
        for mode in range(5):
            for n in (1, 9, 4095, (1 << 17) + 3):
                ZG._check(W, mode, n, seed=n % 97 + W)
            ZG._check(W, mode, 50_001, seed=5, one_segment=True)

    _ran_in_child("test_reduce_scatter", dict(world=W), sweep, K.assigned_to("test_reduce_scatter", world=W), f"W={W}")


@pytest.mark.parametrize("world", WORLDS)
def test_fused_step(world):
    """reduce_scatter_step_ in modes 0, 1, 3 with SGD (with and without momentum), Adam and AdamW, and the bf16-master step,
    bit for bit against torch's fused optimizers on the same reduced shard; one block larger than a stage region."""
    W = world

    def sweep():
        for mode in (0, 1, 3):
            for kind in ("sgd", "sgd0", "adam", "adamw"):
                for n in (9, 4095, (1 << 17) + 3):
                    ZO._check(W, mode, n, kind, seed=n % 89 + W)
        for kind in ("sgd", "sgd0", "adam", "adamw"):
            for n in (9, 4095, (1 << 17) + 3):
                ZM._check(W, n, kind, seed=n % 89 + W)
        mode, kind = ((0, "sgd"), (1, "adamw"), (3, "adam"))[W % 3]
        n = 6_000_003  # stage_mb=8: several launches along the block axis
        assert ZO.Z.padded_block(n, W) * (4 if mode == 1 else 2) > (8 << 20) // (W + 1)
        ZO._check(W, mode, n, kind, seed=3, n_steps=2)

    _ran_in_child("test_fused_step", dict(world=W), sweep, K.assigned_to("test_fused_step", world=W), f"W={W}")


@pytest.mark.parametrize("world", WORLDS)
def test_reduce(world):
    """reduce_ at every root, float and exact, against the oracles and allreduce_op_; other ranks and guards untouched;
    stage_mb=1 with the launch count checked."""
    W = world

    def sweep():
        w = World([0] * W)
        try:
            for dtype, ops in EX.OPS.items():
                for op in ops:
                    for root in range(W):
                        for i, n in enumerate((9, (1 << 17) + 3)):
                            RD.check_reduce(w, dtype, op, n, seed=10 * i + root, root=root, against_allreduce=root == W - 1)
                    RD.check_reduce(w, dtype, op, 1, seed=5, root=0, against_allreduce=False)
                    RD.check_reduce(w, dtype, op, 4095, seed=6, root=W - 1, offset=1)
        finally:
            w.close()
        w = World([0] * W, stage_mb=1)
        slice_cap = ((1 << 20) // (W + 1)) & ~255
        try:
            for dtype in EX.OPS:
                per_elem = {"float32": 4, "int32": 4, "int64": 8}.get(dtype, 2)
                cap = W * (slice_cap // per_elem)
                n = 2 * cap + cap // 3 + 5
                before = w.comms[0].launches
                RD.check_reduce(w, dtype, "sum", n, seed=7, root=W // 2, offset=1, against_allreduce=False)
                assert w.comms[0].launches - before == -(-n // cap) >= 3, dtype
        finally:
            w.close()

    _ran_in_child("test_reduce", dict(world=W), sweep, K.assigned_to("test_reduce", world=W), f"W={W}")


@pytest.mark.parametrize("world", WORLDS)
def test_runtime_world_kernels(world):
    """The kernels whose world is a run-time value, at these worlds: allreduce_op_, allgather_, alltoall_, broadcast_,
    barrier and batchnorm_stats_."""
    W = world

    def sweep():
        w = World([0] * W)
        try:
            for dtype, ops in EX.OPS.items():
                for op in ops:
                    EX.check_reduce(w, dtype, op, 9, seed=1)
                    EX.check_reduce(w, dtype, op, 4095, seed=2, offset=1)
            for dtype in EX.TORCH:
                EX.check_gather(w, dtype, 4095, seed=3, in_off=3, out_off=1)
                EX.check_gather(w, dtype, 9, seed=4, in_place=True)
            for dtype in AA.DTYPES:
                e = AA._esize(dtype)
                for seed in range(2):
                    rng = np.random.default_rng(100 * W + seed)
                    counts = AA._random_counts(rng, W, e, idle=seed if seed else None)
                    x = AA.Exchange(w, dtype, counts, seed=seed)
                    w.run(x.call)
                    x.check()
            for nbytes, root, off in ((1, 0, 0), (4096, W - 1, 0), (100003, 2, 1)):
                src = np.random.default_rng(nbytes).integers(0, 256, size=nbytes + off, dtype=np.uint8)
                tens = [torch.from_numpy((src if r == root else np.full(nbytes + off, r, np.uint8)).copy()).to("cuda:0")[off:]
                        for r in range(W)]
                w.run(lambda r, c, s: c.broadcast_(tens[r], root=root, stream=s))
                for r in range(W):
                    assert np.array_equal(tens[r].cpu().numpy(), src[off:]), (nbytes, root, r)
            w.run(lambda r, c, s: c.barrier(stream=s))
            for k, counts in enumerate(SB.count_patterns(W)):
                SB.check_stats(w, (3, 2048)[k % 2], counts, running=(k % 2 == 0, True), momentum=0.1, eps=1e-5, off=k % 3, seed=k)
        finally:
            w.close()

    want = {"k_allgather", "k_alltoall", "k_broadcast", "k_barrier", "k_bn_stats"}
    want |= {f"k_reduce_exact<{d}, {o}>" for d, o in K.EXACT}
    _ran_in_child("test_runtime_world_kernels", dict(world=W), sweep, want, f"W={W}")


# C = 2056: 257 vecs, two column tiles, the last holding one vec; 4096: two full tiles; 4104: three tiles, the last holding
# one vec, with M = 2 (one CTA row, no merge of ATen's CTA rows) and M = 2048 (grid_y = 8: the merge kernels run)
BN_SHAPES = [(4, 2056, 3, 5), (8, 2056, 16, 16), (2, 4096, 4, 4), (2, 4104, 1, 1), (8, 4104, 16, 16)]


def _bn_geometry(shape):
    """(column tiles of the elementwise passes, vecs in the last one if it is partial, ATen's grid_y of the reductions)."""
    n, c, h, w = shape
    geom, ws = (ctypes.c_int * 4)(), ctypes.c_size_t()
    N.check(N.lib().b2_bn_reduce_plan(n * h * w, c, geom, ctypes.byref(ws)))
    cv = c // 8
    cw = min(cv, 256)  # bn::plan's tile width: kBnThreads vecs
    return -(-cv // cw), cv % cw, geom[3]


def test_batchnorm_column_tiles():
    """The converted BatchNorm2d bit for bit against nn.BatchNorm2d (y, dx, weight and bias gradients, saved and running
    statistics) where the elementwise passes tile the channels in more than one column tile."""
    tiles = {s: _bn_geometry(s) for s in BN_SHAPES}
    assert [t[:2] for t in tiles.values()] == [(2, 1), (2, 1), (2, 0), (3, 1), (3, 1)], tiles
    assert [t[2] for t in tiles.values()] == [1, 8, 1, 1, 8], tiles

    def sweep():
        for i, shape in enumerate(BN_SHAPES):
            BN._run(shape, torch.bfloat16, seed=40 + i)

    _ran_in_child("test_batchnorm_column_tiles", {}, sweep, K.assigned_to("test_batchnorm_column_tiles"), "BatchNorm2d")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("algo", ["oneshot", "twoshot", "twoshot_pipe", "twoshot_ll", "nvls", "auto"])
def test_across_devices(world, algo, cuda_count):
    """One rank per device, as test_allreduce_gpu.py's across-devices case, at W = 5, 6, 7 (skipped on a box with fewer
    GPUs); NVLS against its one-ulp contract where the box has multicast."""
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    w = World(list(range(world)), stage_mb=64)
    try:
        if algo == "nvls" and not w.comms[0].has_multicast:
            pytest.skip("no NVSwitch multicast on this box")
        for c in w.comms:
            c.set_param("pipe_chunk_bytes", 64 << 10)
            c.set_param("nvls_min_bytes", 64 << 10)
            c.set_param("pipe_min_bytes", 256 << 10)
        for mode in ALL_MODES:
            if algo == "nvls" and mode == "f32":
                continue  # fp32-wire NVLS: the switch's fp32 summation order (tools/nvls_probe.py)
            for n in (9, 4099, (1 << 20) + 5):
                _flat(w, n, mode, algo, "special", seed=n)
            _flat(w, (1 << 20) + 5, mode, algo, "nanbits", seed=3)
            if algo == "nvls":
                assert w.comms[0].last_algo == "nvls"
    finally:
        w.close()
