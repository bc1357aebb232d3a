"""b2_reduce_scatter on the GPU: rank r's output against block r of the allreduce oracles (tests/_exact_oracle.py and the
float sum oracles) and against allreduce_op_ of the same inputs on the same communicator, bit for bit; every dtype and op,
W = 1 .. 8 ranks on one device, misaligned buffers with guard bands, the in-place form, blocks cut into several launches;
interleaved with the other collectives; the torch.distributed-shaped helpers under init_pg("b200") in two processes; and
across real devices, next to NCCL's reduce_scatter_tensor at W = 2 (skipped on a box with fewer GPUs)."""
import ctypes
import os
import socket
import subprocess
import sys
import uuid

import numpy as np
import pytest
import torch

import oracle
from tests import _exact_oracle as X
from tests._util import GUARD, World, assert_bits_equal
from tests.test_exact_ops_gpu import (OPS, assert_float_sum_equal, assert_guards, float_sum_oracle, make_inputs, padded,
                                      to_dev, to_host)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [0, 1, 7, 8, 9, 4095, (1 << 17) + 3]  # elements per rank: `in` holds W times as many


def want_block(dtype, op, xs, r, n):
    """Block r of what b2_allreduce_op leaves on every rank, from the oracles."""
    W = len(xs)
    if W == 1:
        return xs[0][r * n:(r + 1) * n]
    if op in ("sum", "avg") and X.is_float(dtype):
        return float_sum_oracle(dtype, xs, 1.0 if op == "sum" else 1.0 / W)[r * n:(r + 1) * n]
    return X.reduce(dtype, op, xs)[r * n:(r + 1) * n]


def assert_oracle_equal(dtype, op, got, want, what):
    if op in ("sum", "avg") and X.is_float(dtype):
        assert_float_sum_equal(dtype, got, want, what)
    else:
        X.assert_exact_equal(dtype, got, want, what)


def check_rs(w, dtype, op, n, seed, in_off=0, out_off=0, in_place=False, against_allreduce=True):
    W = len(w.comms)
    xs = make_inputs(dtype, W, W * n, seed)
    ins, outs = [], []  # (view given to the call, whole allocation, host copy of the allocation before the call)
    for r, c in enumerate(w.comms):
        hi = padded(xs[r], dtype, in_off, GUARD)
        ti = to_dev(hi, dtype, c.device)
        ins.append((ti[in_off:in_off + W * n], ti, hi))
        if in_place:
            outs.append((ti[in_off + r * n:in_off + (r + 1) * n], ti, hi))
        else:
            ho = padded(np.zeros(n, xs[r].dtype), dtype, out_off, GUARD)
            to = to_dev(ho, dtype, c.device)
            outs.append((to[out_off:out_off + n], to, ho))
    w.run(lambda r, c, s: c.reduce_scatter_(outs[r][0], ins[r][0], op, stream=s))
    what = f"reduce_scatter W={W} {dtype} {op} n={n} in_off={in_off} out_off={out_off} in_place={in_place}"
    got = [to_host(o[0], dtype) for o in outs]
    for r in range(W):
        assert_oracle_equal(dtype, op, got[r], want_block(dtype, op, xs, r, n), f"{what} rank={r}")
        whole = to_host(outs[r][1], dtype)
        lo = (in_off + r * n) if in_place else out_off
        assert_guards(whole, outs[r][2], lo, lo + n, f"{what} rank={r}: outside `out`")
        if not in_place:  # the input is only read
            assert np.array_equal(to_host(ins[r][1], dtype).view(np.uint8), ins[r][2].view(np.uint8)), f"{what} rank={r}: input changed"
    if against_allreduce and W > 1 and n:
        # allreduce_op_ of the same inputs on the same communicator: block r is the same bits, NaN payloads included
        full = [to_dev(x, dtype, c.device) for x, c in zip(xs, w.comms)]
        w.run(lambda r, c, s: c.allreduce_op_(full[r], op, stream=s))
        if not (op in ("sum", "avg") and X.is_float(dtype) and w.comms[0].last_algo == "nvls"):  # the switch's order
            for r in range(W):
                ar = to_host(full[r], dtype)[r * n:(r + 1) * n]
                assert np.array_equal(got[r].view(np.uint8), ar.view(np.uint8)), f"{what} rank={r}: differs from allreduce_op_"


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_reduce_scatter_matches_oracle_and_allreduce_one_device(world):
    w = World([0] * world)
    try:
        for dtype, ops in OPS.items():
            for op in ops:
                for i, n in enumerate(SIZES):
                    check_rs(w, dtype, op, n, seed=i)
                check_rs(w, dtype, op, 4095, seed=50, in_off=1, out_off=3)  # misaligned by one / three elements
                check_rs(w, dtype, op, 9, seed=51, in_off=3, out_off=1)
                check_rs(w, dtype, op, 4095, seed=52, in_place=True)
                check_rs(w, dtype, op, 4093, seed=53, in_off=1, in_place=True)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3, 8])
def test_reduce_scatter_chunked(world):
    """stage_mb=1: a recv region holds 1 MiB / (W + 1), so every block is cut into at least 3 launches (the launch count
    is checked), each block's own boundary falling inside a vec."""
    w = World([0] * world, stage_mb=1)
    slice_cap = ((1 << 20) // (world + 1)) & ~255
    n = 3 * (slice_cap // 2) + 5  # > 3 regions of 16-bit elements, more for wider ones
    try:
        for dtype, ops in OPS.items():
            for op in ops:
                per_elem = {"float32": 4, "int32": 4, "int64": 8}.get(dtype, 2)  # stage bytes per element (fp32 wire: 4)
                cap = slice_cap // per_elem
                before = w.comms[0].launches
                check_rs(w, dtype, op, n, seed=7, in_off=1, out_off=3, against_allreduce=False)
                launches = w.comms[0].launches - before
                assert launches == -(-n // cap) >= 3, (dtype, op, launches)
                check_rs(w, dtype, op, n, seed=8, in_place=True, against_allreduce=op in ("sum", "max"))
    finally:
        w.close()


def test_argument_validation_with_a_communicator():
    """The checks that need a communicator: null buffers, and an `out` that overlaps `in` anywhere but this rank's block.
    Nothing is launched, so the other rank does not take part."""
    from torchx_b200.ddp import _native as N

    w = World([0] * 2)
    try:
        L, c = N.lib(), w.comms[1]  # rank 1: its block is in[n:2n]
        buf = torch.zeros(256, dtype=torch.float32, device="cuda:0")
        base = buf.data_ptr()
        for o, i in ((None, base), (base, None), (None, None)):
            assert L.b2_reduce_scatter(c._h, o, i, 8, N.B2_DT_FLOAT32, N.B2_OP_SUM, None) == N.B2_EINVAL
            assert b"b2_reduce_scatter: null buffer" in L.b2_last_error()
        n = 16  # elements per block, 64 bytes
        for out_at in (0, 1, n - 1, n + 1, 2 * n - 1, -n + 1, -1):  # overlaps rank 0's block, straddles, or ends inside `in`
            rc = L.b2_reduce_scatter(c._h, ctypes.c_void_p(base + 256 + 4 * out_at), ctypes.c_void_p(base + 256), n,
                                     N.B2_DT_FLOAT32, N.B2_OP_SUM, None)
            assert rc == N.B2_EINVAL, out_at
            assert b"`out` overlaps `in` other than as this rank's block" in L.b2_last_error(), out_at
        assert w.comms[0].launches == 0 and c.launches == 0
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_interleaved_with_the_other_collectives(world):
    """30 rounds of reduce_scatter_ (exact and float), allreduce_, allreduce_op_, allgather_, broadcast_ and barrier issued
    back to back without a host sync: every op takes the next stage parity and flag sequence number, whatever its kind."""
    w = World([0] * world)
    rounds, n = 30, 1000
    try:
        plan = []
        for k in range(rounds):
            b = [np.random.default_rng(1000 * k + r).standard_normal(n).astype(np.float32) for r in range(world)]
            ints = make_inputs("int64", world, n, seed=k)
            rsi = make_inputs("int64", world, world * 333, seed=k + 300)
            rsf = make_inputs("bfloat16", world, world * 517, seed=k + 700)
            gat = make_inputs("int32", world, 37, seed=k + 500)
            root = k % world
            bc = [np.full(n + 3, (r + 10 * k) % 256, np.uint8) for r in range(world)]
            op = ("sum", "min", "max")[k % 3]
            plan.append(dict(b=b, ints=ints, rsi=rsi, rsf=rsf, gat=gat, root=root, bc=bc, op=op,
                             tb=[torch.from_numpy(x.copy()).cuda() for x in b],
                             ti=[to_dev(x, "int64", 0) for x in ints],
                             trsi=[to_dev(x, "int64", 0) for x in rsi],
                             trsio=[torch.empty(333, dtype=torch.int64, device="cuda:0") for _ in range(world)],
                             trsf=[to_dev(x, "bfloat16", 0) for x in rsf],
                             tg=[to_dev(x, "int32", 0) for x in gat],
                             tgo=[torch.empty(world * 37, dtype=torch.int32, device="cuda:0") for _ in range(world)],
                             tc=[torch.from_numpy(x.copy()).cuda() for x in bc]))
        torch.cuda.synchronize()

        def ops(r, c, s, p):
            return [lambda: c.reduce_scatter_(p["trsio"][r], p["trsi"][r], p["op"], stream=s),
                    lambda: c.allreduce_(p["tb"][r], wire="bf16", stream=s),
                    lambda: c.reduce_scatter_(p["trsf"][r][r * 517:(r + 1) * 517], p["trsf"][r], "sum", stream=s),  # in place
                    lambda: c.allreduce_op_(p["ti"][r], p["op"], stream=s),
                    lambda: c.allgather_(p["tgo"][r], p["tg"][r], stream=s),
                    lambda: c.barrier(stream=s),
                    lambda: c.broadcast_(p["tc"][r], root=p["root"], stream=s)]

        # Every rank here is launched from one host thread, rank 0's whole sequence first.  The first launch of a kernel
        # that CUDA has not loaded yet (lazy module loading) waits for the device, i.e. for rank 0's collective that is
        # already spinning on rank 1 - whose launches this thread has not issued.  So every kernel of the sequence is
        # loaded first, one synchronised op at a time, on scratch copies of rounds 0-2 (SUM, MIN and MAX).
        for p0 in plan[:3]:
            scratch = {k: ([t.clone() for t in v] if k.startswith("t") else v) for k, v in p0.items()}
            for o in range(7):
                w.run(lambda r, c, s: ops(r, c, s, scratch)[o]())

        def issue(r, c, s):
            for p in plan:
                for op in ops(r, c, s, p):
                    op()

        w.run(issue)
        for k, p in enumerate(plan):
            wb = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, p["b"], 1.0 / world)
            wi = X.reduce("int64", p["op"], p["ints"])
            wrsi = X.reduce("int64", p["op"], p["rsi"])
            wrsf = float_sum_oracle("bfloat16", p["rsf"], 1.0)
            wg = X.allgather(p["gat"])
            for r in range(world):
                assert_bits_equal(p["tb"][r].cpu().numpy(), wb, f"round {k} bucket rank {r}")
                assert np.array_equal(to_host(p["ti"][r], "int64"), wi), f"round {k} {p['op']} rank {r}"
                assert np.array_equal(to_host(p["trsio"][r], "int64"), wrsi[r * 333:(r + 1) * 333]), f"round {k} rs {p['op']} rank {r}"
                got_f = to_host(p["trsf"][r], "bfloat16")
                assert_float_sum_equal("bfloat16", got_f[r * 517:(r + 1) * 517], wrsf[r * 517:(r + 1) * 517], f"round {k} rs bf16 rank {r}")
                others = np.delete(got_f, np.s_[r * 517:(r + 1) * 517])
                assert np.array_equal(others, np.delete(p["rsf"][r], np.s_[r * 517:(r + 1) * 517])), f"round {k} rs bf16 rank {r}: input"
                assert np.array_equal(to_host(p["tgo"][r], "int32").view(np.uint8), wg), f"round {k} gather rank {r}"
                assert np.array_equal(p["tc"][r].cpu().numpy(), p["bc"][p["root"]]), f"round {k} broadcast rank {r}"
    finally:
        w.close()


def _run_workers(tmp_path, world, devices, backend, port=0):
    shm = f"/b2_rs_{uuid.uuid4().hex[:12]}"
    procs = []
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "reduce_scatter_worker.py"), "--rank", str(r), "--world",
               str(world), "--device", str(devices[r]), "--shm", shm, "--out", str(tmp_path / f"r{r}.npz"), "--backend", backend,
               "--port", str(port)]
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
        assert p.returncode == 0, f"rank {r} failed:\n{outs[r]}"
    return [dict(np.load(tmp_path / f"r{r}.npz")) for r in range(world)]


def test_public_helpers_two_processes_one_gpu(tmp_path):
    """Two worker processes on cuda:0 under init_pg("b200") (tests/workers/reduce_scatter_worker.py)."""
    W = 2
    got = _run_workers(tmp_path, W, [0] * W, "b200")
    for r in range(W):
        g = got[r]
        assert g["rs_tensor_sum"].tolist() == [(r + 1) * W * (W + 1) // 2] * 3
        m = g["rs_tensor_max"]
        if r == 0:
            assert m[0] == 1.0 and m[1] == 0.0 and np.signbit(m[1])  # max(-0.0, -1.0) = -0.0
        else:
            assert m[0] == 0.5 and np.isnan(m[1])
        a = g["rs_tensor_avg"]
        if r == 0:
            assert a.tolist() == [0.5, -0.5]
        else:
            assert a[0] == 0.25 and np.isnan(a[1])
        base = np.arange(4).reshape(2, 2) * (r + 1)
        assert g["rs_list_sum"].tolist() == (W * base + 100 * W * (W - 1) // 2).tolist()
        assert g["rs_list_min"].tolist() == base.tolist()
        assert g["broadcast"].tolist() == [1001, 7]
        assert g["broadcast_bf16"].tolist() == [1.0] * 5


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
                    check_rs(w, dtype, op, n, seed=n)
                check_rs(w, dtype, op, 4095, seed=1, in_off=1, out_off=3)
                check_rs(w, dtype, op, 4095, seed=2, in_place=True)
    finally:
        w.close()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_equals_nccl_reduce_scatter_at_two_gpus(tmp_path, cuda_count):
    """At W = 2 a float sum is one add and one rounding, so NCCL's reduce_scatter_tensor gives the same bits; integer SUM
    and MIN / MAX of values without NaNs are exact in both (one GPU per rank: skipped on a box with fewer than two)."""
    if cuda_count < 2:
        pytest.skip("needs 2 GPUs")
    got = _run_workers(tmp_path, 2, [0, 1], "nccl", port=_free_port())
    for r in range(2):
        assert got[r]["nccl_bit_equal"].all(), (r, got[r]["nccl_bit_equal"])
