"""The exact collectives on the GPU: b2_allreduce_op (integer SUM, MIN / MAX on every dtype, float SUM / AVG through the
gradient allreduce) and b2_allgather, bit for bit against tests/_exact_oracle.py and the sum oracles, with guard bands,
misaligned pointers and messages cut into several launches; interleaved with the other collectives on one communicator;
and the torch.distributed-shaped helpers under init_pg("b200") in two processes."""
import ctypes
import os
import subprocess
import sys
import uuid

import numpy as np
import pytest
import torch

import oracle
from tests import _exact_oracle as X
from tests import _oracle_f16 as F16
from tests._util import GUARD, World, assert_bits_equal, assert_guards_intact

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TORCH = {"int32": torch.int32, "int64": torch.int64, "float32": torch.float32, "bfloat16": torch.bfloat16,
         "float16": torch.float16, "uint8": torch.uint8}
SIGNED = {np.uint32: torch.int32, np.uint16: torch.int16}  # how raw float bits travel to and from torch
OPS = {"int32": ["sum", "min", "max"], "int64": ["sum", "min", "max"],
       "float32": ["sum", "avg", "min", "max"], "bfloat16": ["sum", "avg", "min", "max"], "float16": ["sum", "avg", "min", "max"]}
SIZES = [0, 1, 7, 8, 9, 4095, (1 << 20) + 3]
POISON = {"int32": 0x5A5A5A5A, "int64": 0x5A5A5A5A5A5A5A5A, "float32": 0x5A5A5A5A, "bfloat16": 0x5A5A, "float16": 0x5A5A,
          "uint8": 0x5A}
SPECIAL_BITS = {
    "float32": [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0xFFFFFFFF, 0x7F800001, 0x00000001,
                0x7F7FFFFF],
    "bfloat16": [0x0000, 0x8000, 0x7F80, 0xFF80, 0x7FC0, 0xFFFF, 0x7F81, 0x0001, 0x7F7F, 0xFF7F],
    "float16": [0x0000, 0x8000, 0x7C00, 0xFC00, 0x7E00, 0xFFFF, 0x7C01, 0x0001, 0x7BFF, 0xFBFF],
}


def host_dtype(dtype):
    return np.uint8 if dtype == "uint8" else X.DTYPES[dtype][0]


def make_inputs(dtype, world, n, seed):
    """Per-rank host buffers: integers with the extremes sprinkled in (so SUM wraps), floats as bit patterns of normal
    values with zeros of both signs, +-inf, NaNs (0xFFFF among them) and subnormals sprinkled in at a low rate."""
    out = []
    for r in range(world):
        rng = np.random.default_rng(seed * 131 + r)
        if dtype in ("int32", "int64", "uint8"):
            info = np.iinfo(host_dtype(dtype))
            x = rng.integers(info.min, info.max, size=n, dtype=host_dtype(dtype), endpoint=True)
            if n and dtype != "uint8":
                idx = rng.integers(0, n, size=max(1, n // 5))
                x[idx] = rng.choice(np.array([info.min, info.max, -1, 0, 1], dtype=x.dtype), size=idx.size)
        else:
            v = rng.standard_normal(n).astype(np.float32)
            if dtype == "float32":
                x = v.view(np.uint32).copy()
            elif dtype == "bfloat16":
                x = oracle.f32_to_bf16_bits(v)
            else:
                x = F16.f32_to_f16_bits(v).copy()
            if n:
                idx = rng.integers(0, n, size=max(1, n // 41))
                x[idx] = rng.choice(np.array(SPECIAL_BITS[dtype], dtype=x.dtype), size=idx.size)
        out.append(np.ascontiguousarray(x))
    return out


def to_dev(h, dtype, device):
    if h.dtype.type in SIGNED:  # raw float bits: through the signed integer type of the same width
        t = torch.from_numpy(h.view(np.int32 if h.dtype == np.uint32 else np.int16).copy())
        return t.to(f"cuda:{device}").view(TORCH[dtype])
    return torch.from_numpy(h.copy()).to(f"cuda:{device}")


def to_host(t, dtype):
    h = host_dtype(dtype)
    if h in SIGNED:
        return t.view(SIGNED[h]).cpu().numpy().view(h)
    return t.cpu().numpy()


def padded(h, dtype, lo, hi):
    fill = np.array([POISON[dtype]], dtype=np.uint64).astype(h.dtype)
    return np.concatenate([np.full(lo, fill[0], h.dtype), h, np.full(hi, fill[0], h.dtype)])


def assert_guards(got, before, lo, hi, what):
    """assert_guards_intact on the 16- or 32-bit words of elements of any width."""
    u = np.uint16 if got.itemsize == 2 else np.uint32
    k = max(1, got.itemsize // 4)
    assert_guards_intact(got.view(u), before.view(u), lo * k, hi * k, what)


def float_sum_oracle(dtype, xs, scale):
    if dtype == "float32":
        return oracle.allreduce(oracle.B2O_F32, [x.view(np.float32) for x in xs], scale).view(np.uint32)
    if dtype == "bfloat16":
        return oracle.allreduce(oracle.B2O_BF16, xs, scale)
    return F16.allreduce(F16.B2O_F16, xs, scale)


def assert_float_sum_equal(dtype, got, want, what):
    if dtype == "float16":
        F16.assert_f16_bits_equal(got, want, what)
    elif dtype == "float32":
        assert_bits_equal(got.view(np.float32), want.view(np.float32), what)
    else:
        assert_bits_equal(got, want, what)


def check_reduce(w, dtype, op, n, seed, offset=0):
    W = len(w.comms)
    xs = make_inputs(dtype, W, n, seed)
    full, tens, before = [], [], []
    for r, c in enumerate(w.comms):
        h = padded(xs[r], dtype, offset, GUARD)
        t = to_dev(h, dtype, c.device)
        full.append(t)
        tens.append(t[offset:offset + n])
        before.append(h)
    w.run(lambda r, c, s: c.allreduce_op_(tens[r], op, stream=s))
    what = f"W={W} {dtype} {op} n={n} off={offset}"
    got = [to_host(f, dtype) for f in full]
    for r in range(W):
        assert_guards(got[r], before[r], offset, offset + n, f"{what} rank={r}")
        assert np.array_equal(got[r][offset:offset + n], got[0][offset:offset + n]), f"{what}: rank {r} differs from rank 0"
    res = got[0][offset:offset + n]
    if W == 1:
        assert np.array_equal(res, xs[0]), f"{what}: W = 1 must leave the buffer as it is"
    elif op in ("sum", "avg") and X.is_float(dtype):
        assert_float_sum_equal(dtype, res, float_sum_oracle(dtype, xs, 1.0 if op == "sum" else 1.0 / W), what)
    else:
        X.assert_exact_equal(dtype, res, X.reduce(dtype, op, xs), what)


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_allreduce_op_matches_oracle_one_device(world):
    w = World([0] * world)
    try:
        for dtype, ops in OPS.items():
            for op in ops:
                for i, n in enumerate(SIZES):
                    check_reduce(w, dtype, op, n, seed=i)
                check_reduce(w, dtype, op, 4095, seed=50, offset=1)  # pointer misaligned by one element
                check_reduce(w, dtype, op, 9, seed=51, offset=3)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3, 8])
def test_allreduce_op_chunked(world):
    """stage_mb=1: a message is cut into several launches (the stage holds 1 MiB / (W + 1) per rank)."""
    w = World([0] * world, stage_mb=1)
    try:
        for dtype, ops in OPS.items():
            for op in ops:
                check_reduce(w, dtype, op, (1 << 18) + 5, seed=7)
                check_reduce(w, dtype, op, (1 << 18) + 5, seed=8, offset=1)
    finally:
        w.close()


def test_float_min_max_nan_and_signed_zero_on_the_gpu():
    """The contract's corner cases spelled out: the .NaN min / max instructions must give a NaN whatever rank holds it, and
    order -0.0 below +0.0 in either rank order."""
    w = World([0] * 3)
    try:
        for dtype, (pz, nz, nan, inf, one) in {"float32": (0, 0x80000000, 0x7FC00000, 0x7F800000, 0x3F800000),
                                                "bfloat16": (0, 0x8000, 0x7FC0, 0x7F80, 0x3F80),
                                                "float16": (0, 0x8000, 0x7E00, 0x7C00, 0x3C00)}.items():
            h = X.DTYPES[dtype][0]
            cols = [[pz, nz, pz], [nz, pz, pz], [pz, pz, nz], [nan, one, one], [one, nan, one], [one, one, nan], [0xFFFF if
                    dtype != "float32" else 0xFFFFFFFF, inf, one], [inf, one, inf | nz], [inf | nz, nz, pz]]
            xs = [np.array([c[r] for c in cols], dtype=h) for r in range(3)]
            for op in ("min", "max"):
                tens = [to_dev(x, dtype, 0) for x in xs]
                w.run(lambda r, c, s: c.allreduce_op_(tens[r], op, stream=s))
                got = [to_host(t, dtype) for t in tens]
                want = X.reduce(dtype, op, xs)
                for r in range(3):
                    assert np.array_equal(got[r], got[0]), (dtype, op, r)
                    X.assert_exact_equal(dtype, got[r], want, f"{dtype} {op} rank={r}")
                zeros = got[0][:3]
                assert (zeros == (nz if op == "min" else pz)).all(), (dtype, op, zeros)
                assert X.isnan_bits(dtype, got[0][3:7]).all(), (dtype, op)
    finally:
        w.close()


def check_gather(w, dtype, n, seed, in_off=0, out_off=0, in_place=False):
    W = len(w.comms)
    xs = make_inputs(dtype, W, n, seed)
    outs, ins = [], []
    for r, c in enumerate(w.comms):
        ho = padded(np.zeros(W * n, xs[r].dtype), dtype, out_off, GUARD)
        to = to_dev(ho, dtype, c.device)
        outs.append((to, ho))
        if in_place:
            to[out_off + r * n:out_off + (r + 1) * n] = to_dev(xs[r], dtype, c.device)
            ho[out_off + r * n:out_off + (r + 1) * n] = xs[r]
            ins.append((to[out_off + r * n:out_off + (r + 1) * n], None))
        else:
            hi = padded(xs[r], dtype, in_off, GUARD)
            ti = to_dev(hi, dtype, c.device)
            ins.append((ti[in_off:in_off + n], (ti, hi)))
    w.run(lambda r, c, s: c.allgather_(outs[r][0][out_off:out_off + W * n], ins[r][0], stream=s))
    what = f"allgather W={W} {dtype} n={n} in_off={in_off} out_off={out_off} in_place={in_place}"
    want = X.allgather(xs)
    for r in range(W):
        got = to_host(outs[r][0], dtype)
        assert np.array_equal(got[out_off:out_off + W * n].view(np.uint8), want), f"{what} rank={r}"
        assert np.array_equal(np.delete(got, np.s_[out_off:out_off + W * n]).view(np.uint8),
                              np.delete(outs[r][1], np.s_[out_off:out_off + W * n]).view(np.uint8)), f"{what} rank={r}: guard"
        if ins[r][1] is not None:  # the input is only read
            ti, hi = ins[r][1]
            assert np.array_equal(to_host(ti, dtype).view(np.uint8), hi.view(np.uint8)), f"{what} rank={r}: input changed"


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_allgather_matches_oracle_one_device(world):
    w = World([0] * world)
    try:
        for dtype in TORCH:
            for i, n in enumerate([0, 1, 7, 9, 4095, (1 << 18) + 3]):
                check_gather(w, dtype, n, seed=i)
            check_gather(w, dtype, 4095, seed=20, in_off=1)
            check_gather(w, dtype, 4095, seed=21, out_off=1)
            check_gather(w, dtype, 4095, seed=22, in_off=3, out_off=1)
            check_gather(w, dtype, 4095, seed=23, in_place=True)
            check_gather(w, dtype, 4095, seed=24, out_off=1, in_place=True)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3])
def test_allgather_chunked(world):
    w = World([0] * world, stage_mb=1)
    try:
        for dtype in ("uint8", "int64", "bfloat16"):
            check_gather(w, dtype, (1 << 19) + 7, seed=3)
            check_gather(w, dtype, (1 << 19) + 7, seed=4, in_off=1, out_off=3)
            check_gather(w, dtype, (1 << 19) + 7, seed=5, in_place=True)
    finally:
        w.close()


def test_argument_validation_with_a_communicator():
    """The checks that need a communicator: null buffers, and an all-gather input that overlaps `out` anywhere but this
    rank's block.  Nothing is launched, so the other rank does not take part."""
    from torchx_b200.ddp import _native as N

    w = World([0] * 2)
    try:
        L, c = N.lib(), w.comms[1]  # rank 1: its block is out[n:2n]
        assert L.b2_allreduce_op(c._h, None, 8, N.B2_DT_INT32, N.B2_OP_SUM, None) == N.B2_EINVAL
        assert b"b2_allreduce_op: null buffer" in L.b2_last_error()
        out = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
        base = out.data_ptr()
        for p in (None, base):
            assert L.b2_allgather(c._h, p, None if p else base, 16, None) == N.B2_EINVAL
            assert b"b2_allgather: null buffer" in L.b2_last_error()
        n = 16
        for in_at in (0, 1, n - 1, n + 1, 2 * n - 1, -n + 1):  # overlaps rank 0's block, straddles, or starts before `out`
            rc = L.b2_allgather(c._h, ctypes.c_void_p(base + 16), ctypes.c_void_p(base + 16 + in_at), n, None)
            assert rc == N.B2_EINVAL, in_at
            assert b"`in` overlaps `out` other than as this rank's block" in L.b2_last_error(), in_at
        assert w.comms[0].launches == 0 and c.launches == 0
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_interleaved_with_the_other_collectives(world):
    """30 rounds of bucket allreduce_, allreduce_op_, allgather_ and broadcast_ issued back to back without a host sync:
    every op takes the next stage parity and flag sequence number after the one before it, whatever its kind."""
    w = World([0] * world)
    rounds, n = 30, 1000
    try:
        plan = []
        for k in range(rounds):
            b = [np.random.default_rng(1000 * k + r).standard_normal(n).astype(np.float32) for r in range(world)]
            ints = make_inputs("int64", world, n, seed=k)
            gat = make_inputs("int32", world, 37, seed=k + 500)
            root = k % world
            bc = [np.full(n + 3, (r + 10 * k) % 256, np.uint8) for r in range(world)]
            op = ("sum", "min", "max")[k % 3]
            plan.append(dict(b=b, ints=ints, gat=gat, root=root, bc=bc, op=op,
                             tb=[torch.from_numpy(x.copy()).cuda() for x in b],
                             ti=[to_dev(x, "int64", 0) for x in ints],
                             tg=[to_dev(x, "int32", 0) for x in gat],
                             tgo=[torch.empty(world * 37, dtype=torch.int32, device="cuda:0") for _ in range(world)],
                             tc=[torch.from_numpy(x.copy()).cuda() for x in bc]))
        torch.cuda.synchronize()

        def ops(r, c, s, p):
            return [lambda: c.allreduce_(p["tb"][r], wire="bf16", stream=s),
                    lambda: c.allreduce_op_(p["ti"][r], p["op"], stream=s),
                    lambda: c.allgather_(p["tgo"][r], p["tg"][r], stream=s),
                    lambda: c.broadcast_(p["tc"][r], root=p["root"], stream=s)]

        # Every rank here is launched from one host thread, rank 0's whole sequence first.  The first launch of a kernel
        # that CUDA has not loaded yet (lazy module loading) waits for the device, i.e. for rank 0's collective that is
        # already spinning on rank 1 - whose launches this thread has not issued.  So every kernel of the sequence is
        # loaded first, one synchronised op at a time, on scratch copies of rounds 0-2 (SUM, MIN and MAX).
        for p0 in plan[:3]:
            scratch = {k: ([t.clone() for t in v] if k.startswith("t") else v) for k, v in p0.items()}
            for o in range(4):
                w.run(lambda r, c, s: ops(r, c, s, scratch)[o]())

        def issue(r, c, s):
            for p in plan:
                for op in ops(r, c, s, p):
                    op()

        w.run(issue)
        for k, p in enumerate(plan):
            wb = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, p["b"], 1.0 / world)
            wi = X.reduce("int64", p["op"], p["ints"])
            wg = X.allgather(p["gat"])
            for r in range(world):
                assert_bits_equal(p["tb"][r].cpu().numpy(), wb, f"round {k} bucket rank {r}")
                assert np.array_equal(to_host(p["ti"][r], "int64"), wi), f"round {k} {p['op']} rank {r}"
                assert np.array_equal(to_host(p["tgo"][r], "int32").view(np.uint8), wg), f"round {k} gather rank {r}"
                assert np.array_equal(p["tc"][r].cpu().numpy(), p["bc"][p["root"]]), f"round {k} broadcast rank {r}"
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_across_devices(world, cuda_count):
    """Real NVLink / NVSwitch peers (skipped on a box with fewer GPUs)."""
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    w = World(list(range(world)), stage_mb=64)
    try:
        for dtype, ops in OPS.items():
            for op in ops:
                for n in (9, 4095, (1 << 20) + 3):
                    check_reduce(w, dtype, op, n, seed=n)
            check_gather(w, dtype, (1 << 20) + 3, seed=1, in_off=1)
            check_gather(w, dtype, 4095, seed=2, in_place=True)
    finally:
        w.close()


def test_public_helpers_two_processes_one_gpu(tmp_path):
    """Two worker processes on cuda:0 under init_pg("b200") (tests/workers/exact_ops_worker.py)."""
    world = 2
    shm = f"/b2_exact_{uuid.uuid4().hex[:12]}"
    procs = []
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "exact_ops_worker.py"), "--rank", str(r), "--world",
               str(world), "--device", "0", "--shm", shm, "--out", str(tmp_path / f"r{r}.npz")]
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
    for r in range(world):
        got = dict(np.load(tmp_path / f"r{r}.npz"))
        assert got["one_hot"].tolist() == [1] * world and int(got["computed_world_size"]) == world
        m = got["max"]
        assert m[0] == world - 0.5 and m[1] == 0.0 and np.isnan(m[2])
        assert m[3] == 0.0 and not np.signbit(m[3])  # max(-0.0, +0.0) = +0.0
        want = np.concatenate([np.arange(5, dtype=np.int32) + 10 * q for q in range(world)])
        assert got["gather_into_tensor"].tolist() == want.tolist()
        assert got["gather_list"].reshape(-1).tolist() == want.tolist()
