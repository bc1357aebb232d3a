"""The exact collectives without a GPU: header against binding, argument validation of b2_allreduce_op / b2_allgather, the
numpy oracle (tests/_exact_oracle.py) against independent restatements of the contract, and the dtype / ReduceOp dispatch
of Communicator.allreduce_op_ and of the torch.distributed-shaped helpers."""
import ctypes
import itertools
import os
import re

import numpy as np
import pytest
import torch
import torch.distributed as dist

from tests import _exact_oracle as X
from torchx_b200.ddp import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32_INF, F32_NINF, F32_NAN, F32_NNAN = 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001


def test_header_constants_match_binding():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    names = [f"B2_DT_{d}" for d in ("INT32", "INT64", "FLOAT32", "BFLOAT16", "FLOAT16")] + \
        [f"B2_OP_{o}" for o in ("SUM", "AVG", "MIN", "MAX")]
    for name in names:
        m = re.search(rf"#define\s+{name}\s+\(?(-?\d+)\)?", src)
        assert m, name
        assert int(m.group(1)) == getattr(N, name), name


def test_argument_validation_without_a_gpu():
    L = N.lib()
    buf = ctypes.c_void_p(4096)
    for dt in (-1, 5, 99):
        assert L.b2_allreduce_op(None, buf, 8, dt, N.B2_OP_SUM, None) == N.B2_EINVAL, dt
        assert f"b2_allreduce_op: unknown dtype {dt}".encode() in L.b2_last_error()
    for op in (-1, 4, 99):
        assert L.b2_allreduce_op(None, buf, 8, N.B2_DT_FLOAT32, op, None) == N.B2_EINVAL, op
        assert f"b2_allreduce_op: unknown op {op}".encode() in L.b2_last_error()
    for dt, name in ((N.B2_DT_INT32, b"int32"), (N.B2_DT_INT64, b"int64")):
        assert L.b2_allreduce_op(None, buf, 8, dt, N.B2_OP_AVG, None) == N.B2_EINVAL
        assert b"AVG needs a floating-point dtype, got " + name in L.b2_last_error()
        assert L.b2_allreduce_op(None, buf, 0, dt, N.B2_OP_AVG, None) == N.B2_EINVAL  # rejected even when empty
    # n == 0: a no-op that reads nothing else
    for dt in range(5):
        assert L.b2_allreduce_op(None, None, 0, dt, N.B2_OP_MAX, None) == N.B2_OK
    assert L.b2_allgather(None, None, None, 0, None) == N.B2_OK
    # null pointers
    assert L.b2_allreduce_op(None, buf, 8, N.B2_DT_INT64, N.B2_OP_SUM, None) == N.B2_EINVAL
    assert b"null communicator" in L.b2_last_error()
    assert L.b2_allgather(None, buf, buf, 16, None) == N.B2_EINVAL
    assert b"null communicator" in L.b2_last_error()
    # (null buffers and overlapping all-gather buffers need a communicator: tests/test_exact_ops_gpu.py)


# ---- the oracle ------------------------------------------------------------------------------------------------------
def test_integer_sum_wraps_at_the_extremes():
    for dtype, bits in (("int32", 32), ("int64", 64)):
        host = X.DTYPES[dtype][0]
        lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
        cases = [[hi, 1], [lo, -1], [hi, hi], [lo, lo], [hi, lo], [-1, 1], [hi, 1, lo, -1, 5], [lo, lo, lo, lo, lo, lo, lo, lo]]
        for c in cases:
            xs = [np.array([v], dtype=host) for v in c]
            want = (sum(c) + (1 << (bits - 1))) % (1 << bits) - (1 << (bits - 1))  # Python ints, reduced mod 2^bits
            assert int(X.reduce(dtype, "sum", xs)[0]) == want, (dtype, c)
            assert int(X.reduce(dtype, "min", xs)[0]) == min(c) and int(X.reduce(dtype, "max", xs)[0]) == max(c), (dtype, c)


def _f32(bits):
    return [np.array([b], dtype=np.uint32) for b in bits]


def test_signed_zeros_in_every_rank_order():
    for dtype, pz, nz in (("float32", 0x00000000, 0x80000000), ("bfloat16", 0x0000, 0x8000), ("float16", 0x0000, 0x8000)):
        host = X.DTYPES[dtype][0]
        for w in (2, 3, 4):
            for order in set(itertools.permutations([nz] + [pz] * (w - 1))) | set(itertools.permutations([pz] + [nz] * (w - 1))):
                xs = [np.array([b], dtype=host) for b in order]
                assert int(X.reduce(dtype, "min", xs)[0]) == nz, (dtype, order)
                assert int(X.reduce(dtype, "max", xs)[0]) == pz, (dtype, order)


def test_nan_at_any_rank_wins():
    for w in (1, 2, 3, 8):
        for at in range(w):
            for nan in (F32_NAN, F32_NNAN, 0xFFFFFFFF, 0x7F800001):
                vals = [0x3F800000 + r for r in range(w)]  # 1.0 + r ulp
                vals[at] = nan
                for op in ("min", "max"):
                    got = X.reduce("float32", op, _f32(vals))
                    assert X.isnan_bits("float32", got)[0], (w, at, hex(nan), op)


def test_infinities_are_ordinary_values():
    one, big = 0x3F800000, 0x7F7FFFFF
    assert X.reduce("float32", "min", _f32([F32_INF, one, big]))[0] == one
    assert X.reduce("float32", "max", _f32([F32_INF, one, big]))[0] == F32_INF
    assert X.reduce("float32", "min", _f32([F32_NINF, F32_INF]))[0] == F32_NINF
    assert X.reduce("float32", "max", _f32([F32_NINF, F32_NINF]))[0] == F32_NINF
    assert X.reduce("float32", "min", _f32([0x80000000, F32_NINF]))[0] == F32_NINF


@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_16bit_patterns_against_float_arithmetic(dtype):
    """Every pair of a set of bit patterns (0xFFFF, both zeros, +-inf, NaNs of both signs, subnormals, the extremes)
    against numpy's minimum / maximum on the exactly widened values, with the signed-zero rule stated on its own."""
    pats = np.array([0xFFFF, 0x0000, 0x8000, 0x0001, 0x8001, 0x3F80, 0xBF80, 0x3C00, 0xBC00, 0x7BFF, 0xFBFF, 0x7F7F, 0xFF7F,
                     0x7F80, 0xFF80, 0x7C00, 0xFC00, 0x7FC0, 0xFFC0, 0x7E00, 0x7C01, 0x7F81, 0x1234, 0x9234], dtype=np.uint16)

    def widen(b):
        with np.errstate(invalid="ignore"):  # signalling NaNs
            if dtype == "bfloat16":
                return (b.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
            return b.view(np.float16).astype(np.float64)

    a = np.repeat(pats, pats.size)
    b = np.tile(pats, pats.size)
    for op, f in (("min", np.minimum), ("max", np.maximum)):
        got = X.reduce(dtype, op, [a, b])
        want = f(widen(a), widen(b))  # propagates NaN
        gv = widen(got)
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(gv), nan), op
        assert np.array_equal(gv[~nan], want[~nan]), op
        both_zero = (widen(a) == 0) & (widen(b) == 0)
        neg = (np.where(op == "min", a | b, a & b) & 0x8000) != 0  # min: -0 if either is -0; max: -0 only if both are
        assert np.array_equal((got[both_zero] & 0x8000) != 0, neg[both_zero]), op
    assert X.isnan_bits(dtype, X.reduce(dtype, "max", [np.array([0xFFFF], np.uint16), np.array([0x7C00], np.uint16)]))[0]


def test_float32_random_against_numpy():
    rng = np.random.default_rng(5)
    xs = [rng.standard_normal(1000).astype(np.float32) for _ in range(5)]
    xs[2][::17] = np.nan
    xs[4][::23] = -np.inf
    bits = [x.view(np.uint32) for x in xs]
    for op, f in (("min", np.minimum), ("max", np.maximum)):
        got = X.reduce("float32", op, bits).view(np.float32)
        want = f.reduce(np.stack(xs), axis=0)
        assert np.array_equal(got, want, equal_nan=True), op


def test_float_sum_is_not_an_exact_op():
    for dtype in ("float32", "bfloat16", "float16"):
        with pytest.raises(ValueError):
            X.reduce(dtype, "sum", [np.zeros(1, X.DTYPES[dtype][0])])


def test_allgather_oracle_is_rank_order_bytes():
    xs = [np.arange(5, dtype=np.uint8) + 10 * r for r in range(3)]
    assert X.allgather(xs).tolist() == [0, 1, 2, 3, 4, 10, 11, 12, 13, 14, 20, 21, 22, 23, 24]


# ---- dispatch --------------------------------------------------------------------------------------------------------
def test_dtype_op_dispatch():
    from torchx_b200.ddp.comm import dtype_op_for

    want_dt = {torch.int32: N.B2_DT_INT32, torch.int64: N.B2_DT_INT64, torch.float32: N.B2_DT_FLOAT32,
               torch.bfloat16: N.B2_DT_BFLOAT16, torch.float16: N.B2_DT_FLOAT16}
    want_op = {"sum": N.B2_OP_SUM, "avg": N.B2_OP_AVG, "min": N.B2_OP_MIN, "max": N.B2_OP_MAX}
    for dt, code in want_dt.items():
        for op, opc in want_op.items():
            if op == "avg" and not dt.is_floating_point:
                with pytest.raises(TypeError, match="avg needs a floating-point tensor"):
                    dtype_op_for(dt, op)
            else:
                assert dtype_op_for(dt, op) == (code, opc)
    for dt in (torch.float64, torch.uint8, torch.int8, torch.int16, torch.bool, torch.complex64):
        with pytest.raises(TypeError, match="unsupported dtype"):
            dtype_op_for(dt, "sum")
    for op in ("product", "band", "bor", "bxor", "premul_sum", "SUM"):
        with pytest.raises(ValueError, match="unsupported op"):
            dtype_op_for(torch.int64, op)


def test_reduce_op_names():
    from torchx_b200.distributed import reduce_op_name

    R = dist.ReduceOp
    assert [reduce_op_name(o) for o in (R.SUM, R.AVG, R.MIN, R.MAX)] == ["sum", "avg", "min", "max"]
    assert reduce_op_name(R(R.MAX)) == "max"  # a ReduceOp instance, not only the enum value
    for o in (R.PRODUCT, R.BAND, R.BOR, R.BXOR):
        with pytest.raises(ValueError, match="supports SUM, AVG, MIN and MAX"):
            reduce_op_name(o)


class _FakeComm:
    """Stands in for the native communicator: records calls; all-gather writes rank r's block as input + 100 r."""

    def __init__(self, world):
        self.world = world
        self.calls = []

    def allreduce_op_(self, t, op):
        self.calls.append(("allreduce_op_", op))
        return t

    def allgather_(self, out, t):
        self.calls.append(("allgather_", out.shape, t.shape))
        for r in range(self.world):
            out.view(self.world, -1)[r].copy_(t.reshape(-1) + 100 * r)
        return out


def test_helpers_run_on_the_native_communicator(monkeypatch):
    import torchx_b200.distributed as D

    assert not dist.is_initialized()
    fake = _FakeComm(3)
    monkeypatch.setattr(D, "_COMM", fake)
    t = torch.arange(4, dtype=torch.int64)
    assert D.all_reduce(t) is None
    assert D.all_reduce(t, op=dist.ReduceOp.MAX, group=dist.group.WORLD) is None
    assert fake.calls == [("allreduce_op_", "sum"), ("allreduce_op_", "max")]
    with pytest.raises(ValueError):
        D.all_reduce(t, op=dist.ReduceOp.PRODUCT)
    with pytest.raises(NotImplementedError, match="no work handles"):
        D.all_reduce(t, async_op=True)
    with pytest.raises(NotImplementedError, match="no subgroups"):
        D.all_reduce(t, group=object())
    out = torch.empty(12, dtype=torch.int64)
    D.all_gather_into_tensor(out, t)
    assert out.tolist() == [0, 1, 2, 3, 100, 101, 102, 103, 200, 201, 202, 203]
    lst = [torch.empty(2, 2, dtype=torch.int64) for _ in range(3)]
    D.all_gather(lst, t.view(2, 2))
    assert [x.reshape(-1).tolist() for x in lst] == [[0, 1, 2, 3], [100, 101, 102, 103], [200, 201, 202, 203]]
    with pytest.raises(ValueError, match="world size is 3"):
        D.all_gather(lst[:2], t)
    with pytest.raises(ValueError, match="every tensor of tensor_list"):
        D.all_gather([torch.empty(4, dtype=torch.int32)] * 3, t)
    for call in (lambda: D.all_gather_into_tensor(out, t, async_op=True), lambda: D.all_gather(lst, t, group=object())):
        with pytest.raises(NotImplementedError):
            call()


def test_helpers_delegate_without_the_native_communicator(monkeypatch):
    import torchx_b200.distributed as D

    seen = []
    monkeypatch.setattr(D, "_COMM", None)
    monkeypatch.setattr(dist, "all_reduce", lambda *a, **k: seen.append(("all_reduce", k["op"], k["async_op"])) or "work")
    monkeypatch.setattr(dist, "all_gather_into_tensor", lambda *a, **k: seen.append(("all_gather_into_tensor",)))
    monkeypatch.setattr(dist, "all_gather", lambda *a, **k: seen.append(("all_gather",)))
    t = torch.zeros(2)
    assert D.all_reduce(t, op=dist.ReduceOp.PRODUCT, async_op=True) == "work"  # torch's own rules apply there
    D.all_gather_into_tensor(torch.zeros(4), t)
    D.all_gather([t, t], t)
    assert seen == [("all_reduce", dist.ReduceOp.PRODUCT, True), ("all_gather_into_tensor",), ("all_gather",)]
