"""b2_reduce on the GPU: the root's tensor against the allreduce oracles (tests/_exact_oracle.py and the float sum oracles)
and against allreduce_op_ of the same inputs on the same communicator, bit for bit; every other rank's tensor and every
guard band unchanged; every dtype and op, every root, W = 1 .. 8 ranks on one device, misaligned buffers, messages cut
into several launches; interleaved with the other collectives; at op counts around 2^29 .. 2^40 (tests/test_op_count_gpu.py's
checks); and across real devices, next to NCCL's reduce at W = 2 (skipped on a box with fewer GPUs)."""
import os
import subprocess
import sys
import uuid

import numpy as np
import pytest
import torch

import oracle
from tests import _exact_oracle as X
from tests import test_op_count_gpu as OC
from tests._util import GUARD, World, assert_bits_equal
from tests.test_exact_ops_gpu import OPS, assert_guards, make_inputs, padded, to_dev, to_host
from tests.test_reduce_scatter_gpu import SIZES, _free_port, assert_oracle_equal, want_block

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check_reduce(w, dtype, op, n, seed, root, offset=0, against_allreduce=True):
    W = len(w.comms)
    xs = make_inputs(dtype, W, n, seed)
    full, tens, before = [], [], []
    for r, c in enumerate(w.comms):
        h = padded(xs[r], dtype, offset, GUARD)
        t = to_dev(h, dtype, c.device)
        full.append(t)
        tens.append(t[offset:offset + n])
        before.append(h)
    w.run(lambda r, c, s: c.reduce_(tens[r], root, op, stream=s))
    what = f"reduce W={W} {dtype} {op} n={n} root={root} off={offset}"
    got = [to_host(f, dtype) for f in full]
    for r in range(W):
        if r == root:
            assert_guards(got[r], before[r], offset, offset + n, f"{what}: root's guard bands")
        else:  # a non-root's tensor is only read
            assert np.array_equal(got[r].view(np.uint8), before[r].view(np.uint8)), f"{what}: rank {r} changed"
    res = got[root][offset:offset + n]
    assert_oracle_equal(dtype, op, res, want_block(dtype, op, xs, 0, n), what)
    if against_allreduce and W > 1 and n:
        again = [to_dev(x, dtype, c.device) for x, c in zip(xs, w.comms)]
        w.run(lambda r, c, s: c.allreduce_op_(again[r], op, stream=s))
        if not (op in ("sum", "avg") and X.is_float(dtype) and w.comms[0].last_algo == "nvls"):  # the switch's order
            ar = to_host(again[root], dtype)
            assert np.array_equal(res.view(np.uint8), ar.view(np.uint8)), f"{what}: differs from allreduce_op_"


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_reduce_matches_oracle_and_allreduce_one_device(world):
    w = World([0] * world)
    try:
        for dtype, ops in OPS.items():
            for op in ops:
                for i, n in enumerate(SIZES):
                    for root in range(world):
                        check_reduce(w, dtype, op, n, seed=10 * i + root, root=root, against_allreduce=n in (9, 4095, SIZES[-1]))
                for root in range(world):
                    check_reduce(w, dtype, op, 4095, seed=50 + root, root=root, offset=1)  # misaligned by one / three elements
                    check_reduce(w, dtype, op, 9, seed=60 + root, root=root, offset=3)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3, 8])
def test_reduce_chunked(world):
    """stage_mb=1: a launch holds W slices of one recv region (1 MiB / (W + 1)), so the message takes at least 3 launches
    (the count is checked), the last one with slices that end inside a vec."""
    w = World([0] * world, stage_mb=1)
    slice_cap = ((1 << 20) // (world + 1)) & ~255
    try:
        for dtype, ops in OPS.items():
            per_elem = {"float32": 4, "int32": 4, "int64": 8}.get(dtype, 2)  # stage bytes per element (fp32 wire: 4)
            cap = world * (slice_cap // per_elem)
            n = 2 * cap + cap // 3 + 5
            for op in ops:
                root = len(op) % world
                before = w.comms[0].launches
                check_reduce(w, dtype, op, n, seed=7, root=root, offset=1, against_allreduce=False)
                launches = w.comms[0].launches - before
                assert launches == -(-n // cap) >= 3, (dtype, op, launches)
                check_reduce(w, dtype, op, n, seed=8, root=world - 1 - root, against_allreduce=op in ("sum", "max"))
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_interleaved_with_the_other_collectives(world):
    """20 rounds of reduce_ (exact and float, the root rotating) between LL-sized and two-shot-sized allreduce_,
    reduce_scatter_, broadcast_ and a p2p_ exchange, issued back to back without a host sync: a non-root that left a
    reduce early must not overwrite its reduced slice before the root has read it."""
    w = World([0] * world)
    rounds, n, big = 20, 1000, 600_003
    try:
        for c in w.comms:  # the LL kernel for the small bucket, the single-pass two-shot for the big one
            c.set_param("oneshot_max_bytes", 0)
            c.set_param("ll_min_bytes", 0)
            c.set_param("ll_max_bytes", 1 << 20)
        plan = []
        for k in range(rounds):
            root = k % world
            op = ("sum", "min", "max")[k % 3]
            ri = make_inputs("int64", world, 3333, seed=k)
            rf = make_inputs("bfloat16", world, 5171, seed=k + 100)
            b = [np.random.default_rng(1000 * k + r).standard_normal(n).astype(np.float32) for r in range(world)]
            bb = [np.random.default_rng(2000 * k + r).standard_normal(big).astype(np.float32) for r in range(world)]
            rs = make_inputs("int32", world, world * 77, seed=k + 300)
            bc = [np.full(n + 3, (r + 10 * k) % 256, np.uint8) for r in range(world)]
            pp = [np.full(123, 7 * r + k, np.int32) for r in range(world)]
            plan.append(dict(root=root, op=op, ri=ri, rf=rf, b=b, bb=bb, rs=rs, bc=bc, pp=pp,
                             tri=[to_dev(x, "int64", 0) for x in ri], trf=[to_dev(x, "bfloat16", 0) for x in rf],
                             tb=[torch.from_numpy(x.copy()).cuda() for x in b], tbb=[torch.from_numpy(x.copy()).cuda() for x in bb],
                             trs=[to_dev(x, "int32", 0) for x in rs],
                             trso=[torch.empty(77, dtype=torch.int32, device="cuda:0") for _ in range(world)],
                             tc=[torch.from_numpy(x.copy()).cuda() for x in bc],
                             tp=[torch.from_numpy(x.copy()).cuda() for x in pp],
                             tpo=[torch.zeros(123, dtype=torch.int32, device="cuda:0") for _ in range(world)]))
        torch.cuda.synchronize()

        def ops(r, c, s, p):
            nxt, prv = (r + 1) % world, (r - 1) % world
            return [lambda: c.reduce_(p["tri"][r], p["root"], p["op"], stream=s),
                    lambda: c.allreduce_(p["tb"][r], wire="bf16", stream=s),
                    lambda: c.reduce_(p["trf"][r], (p["root"] + 1) % world, "sum", stream=s),
                    lambda: c.reduce_scatter_(p["trso"][r], p["trs"][r], p["op"], stream=s),
                    lambda: c.allreduce_(p["tbb"][r], wire="bf16", stream=s),
                    lambda: c.p2p_([("send", p["tp"][r], nxt), ("recv", p["tpo"][r], prv)], stream=s),
                    lambda: c.broadcast_(p["tc"][r], root=p["root"], stream=s)]

        # load every kernel of the sequence first, one synchronised op at a time, on scratch copies of rounds 0-2 (a
        # kernel's first launch waits for the device, i.e. for a rank already spinning on ranks not launched yet)
        for p0 in plan[:3]:
            scratch = {k: ([t.clone() for t in v] if k.startswith("t") else v) for k, v in p0.items()}
            for o in range(7):
                w.run(lambda r, c, s: ops(r, c, s, scratch)[o]())
        algos = set()
        w.run(lambda r, c, s: [op() for p in plan for op in ops(r, c, s, p)])
        for k, p in enumerate(plan):
            root, froot = p["root"], (p["root"] + 1) % world
            wi = X.reduce("int64", p["op"], p["ri"])
            wf = want_block("bfloat16", "sum", p["rf"], 0, 5171)
            wb = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, p["b"], 1.0 / world)
            wbb = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, p["bb"], 1.0 / world)
            wrs = X.reduce("int32", p["op"], p["rs"])
            for r in range(world):
                gi = to_host(p["tri"][r], "int64")
                assert np.array_equal(gi, wi if r == root else p["ri"][r]), f"round {k} reduce {p['op']} rank {r}"
                gf = to_host(p["trf"][r], "bfloat16")
                if r == froot:
                    assert_oracle_equal("bfloat16", "sum", gf, wf, f"round {k} reduce bf16 rank {r}")
                else:
                    assert np.array_equal(gf, p["rf"][r]), f"round {k} reduce bf16 rank {r}: input changed"
                assert_bits_equal(p["tb"][r].cpu().numpy(), wb, f"round {k} LL bucket rank {r}")
                assert_bits_equal(p["tbb"][r].cpu().numpy(), wbb, f"round {k} two-shot bucket rank {r}")
                assert np.array_equal(to_host(p["trso"][r], "int32"), wrs[r * 77:(r + 1) * 77]), f"round {k} rs rank {r}"
                assert np.array_equal(p["tpo"][r].cpu().numpy(), p["pp"][(r - 1) % world]), f"round {k} p2p rank {r}"
                assert np.array_equal(p["tc"][r].cpu().numpy(), p["bc"][root]), f"round {k} broadcast rank {r}"
        for c in w.comms:
            algos.add(c.last_algo)
        assert algos == {"twoshot"}, algos
    finally:
        w.close()


# ---- op counts: tests/test_op_count_gpu.py's three checks for reduce_ ----------------------------------------------------
def _reduce_case(w):
    W = len(w.comms)
    check_reduce(w, "float32", "sum", 100_003, seed=3, root=W - 1, offset=1, against_allreduce=False)
    check_reduce(w, "int64", "max", 100_003, seed=4, root=0, offset=1, against_allreduce=False)


@pytest.mark.parametrize("base", OC.BASES, ids=OC._ids(OC.BASES))
@pytest.mark.parametrize("world", OC.WORLDS)
def test_op_count_never_written_slots(world, base):
    w = OC._world(world, base)
    try:
        _reduce_case(w)
        OC._counted(w, base)
    finally:
        w.close()


@pytest.mark.parametrize("base", OC.BASES, ids=OC._ids(OC.BASES))
@pytest.mark.parametrize("world", OC.WORLDS)
def test_op_count_aged_slots(world, base):
    """Grid 8: slots 0-7 hold this op's sequence numbers; the next op starts 2^29 + 1 operations later."""
    w = OC._world(world, base, max_ctas=8)
    try:
        _reduce_case(w)
        later, before = base + 2**29 + 1, w.comms[0].launches
        for c in w.comms:
            c.set_param("op_count", later)
        _reduce_case(w)
        OC._counted(w, later, before)
    finally:
        w.close()


@pytest.mark.parametrize("root", ["root", "non-root"])
@pytest.mark.parametrize("base", OC.SOLO_BASES, ids=OC._ids(OC.SOLO_BASES))
@pytest.mark.parametrize("world", OC.WORLDS)
def test_op_count_no_rank_finishes_alone(world, base, root):
    """Rank 0 launched alone keeps waiting for SOLO_S, whether it is the root or not, then completes with the others."""
    w = OC._world(world, base)
    try:
        check_reduce(OC._RankZeroFirst(w), "float32", "sum", 100_003, seed=5, root=0 if root == "root" else world - 1,
                     against_allreduce=False)
        OC._counted(w, base)
    finally:
        w.close()


# ---- processes ---------------------------------------------------------------------------------------------------------------
def _run_workers(tmp_path, world, devices, backend, port=0):
    shm = f"/b2_rd_{uuid.uuid4().hex[:12]}"
    procs = []
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "reduce_objects_worker.py"), "--rank", str(r), "--world",
               str(world), "--device", str(devices[r]), "--shm", shm, "--out", str(tmp_path / f"{backend}{r}.pkl"), "--backend",
               backend, "--port", str(port)]
        procs.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            o, _ = p.communicate(timeout=300)
            outs.append(o)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, p in enumerate(procs):
        assert p.returncode == 0, f"rank {r} ({backend}) failed:\n{outs[r]}"
    import pickle

    return [pickle.load(open(tmp_path / f"{backend}{r}.pkl", "rb")) for r in range(world)]


@pytest.mark.parametrize("world", [2, 4, 8])
def test_across_devices(world, cuda_count):
    """Real NVLink / NVSwitch peers (skipped on a box with fewer GPUs)."""
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    w = World(list(range(world)), stage_mb=64)
    try:
        for dtype, ops in OPS.items():
            for op in ops:
                for n in (9, 4095, (1 << 17) + 3):
                    check_reduce(w, dtype, op, n, seed=n, root=n % world)
                check_reduce(w, dtype, op, 4095, seed=1, root=world - 1, offset=1)
    finally:
        w.close()


def test_equals_nccl_reduce_at_two_gpus(tmp_path, cuda_count):
    """At W = 2 a float sum is one add and one rounding, so NCCL's reduce gives the same bits; integer SUM and MIN / MAX of
    values without NaNs are exact in both (one GPU per rank: skipped on a box with fewer than two)."""
    if cuda_count < 2:
        pytest.skip("needs 2 GPUs")
    got = _run_workers(tmp_path, 2, [0, 1], "nccl", port=_free_port())
    for r in range(2):
        assert all(got[r]["nccl_bit_equal"].values()), (r, got[r]["nccl_bit_equal"])
