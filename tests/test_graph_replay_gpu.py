"""Every collective, the native BatchNorm2d passes and a whole mini-DDP training step, captured in CUDA graphs and replayed.

The data plane keeps its state on the device (DESIGN.md 2.1): stage parity, flag sequence numbers and the LL flow-control
target come from the device op counter, the point-to-point chunk counters are device words, and every table travels by
value in the kernel parameters.  Eager launches cannot tell that apart from a host-side shadow of the same state, since
host and device advance together; a replay can.  So each graph here is replayed several times with fresh data in its
static inputs, with eager work in between, and every replay is checked bit for bit against the oracles.

Capture uses torch's default capture_error_mode="global": a synchronous copy, a stream or event sync or a pageable copy
in a launch path fails the capture.  Each sequence runs once eagerly before capture, so lazy module loading never happens
while peers spin, and the ranks' graphs are captured one after the other (a capture launches nothing).  The communicators
keep World's short timeout: a replay that waits for a peer that never comes ends in B2_ETIMEOUT, not a hang.

What a replay does not advance: ``launches`` and ``last_algo`` are host counters of the calls that launched, so they count
the capture once and stand still over the replays."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch import nn

import oracle
from tests import _exact_oracle as X
from tests import _oracle_f16 as F16
from tests._util import GUARD, World
from torchx_b200.ddp import _native as N

pytestmark = pytest.mark.gpu

REPLAYS = 6
WIRE_MODES = {0: ("f32", "bf16"), 1: ("f32", "f32"), 2: ("bf16", "bf16"), 3: ("f32", "f16"), 4: ("f16", "f16")}
TORCH_DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16, "u8": torch.uint8, "i32": torch.int32,
            "i64": torch.int64}
NP_BITS = {"f32": np.uint32, "bf16": np.uint16, "f16": np.uint16, "u8": np.uint8, "i32": np.int32, "i64": np.int64}
GUARD_BYTE = 0x5A  # guard bands: 0x5A5A5A5A is a finite fp32, 0x5A5A a finite bf16 / fp16


class Buf:
    """``n`` elements of ``kind`` at element offset ``off`` of an allocation with GUARD elements of guard band on either
    side.  ``fill`` writes the guards and new contents; ``read`` checks the guards and returns the contents as bits."""

    def __init__(self, n, kind, off=0):
        self.n, self.kind = n, kind
        self.es = np.dtype(NP_BITS[kind]).itemsize
        self.alloc = torch.empty(2 * GUARD + off + n, dtype=TORCH_DT[kind], device="cuda")
        self.lo = GUARD + off
        self.t = self.alloc[self.lo:self.lo + n]
        self.img = np.full(self.alloc.numel() * self.es, GUARD_BYTE, np.uint8)

    def fill(self, bits):
        bits = np.ascontiguousarray(bits, dtype=NP_BITS[self.kind])
        assert bits.size == self.n
        self.img[self.lo * self.es:(self.lo + self.n) * self.es] = bits.view(np.uint8)
        self.alloc.view(torch.uint8).copy_(torch.from_numpy(self.img))

    def read(self, what):
        got = self.alloc.view(torch.uint8).cpu().numpy()
        a, b = self.lo * self.es, (self.lo + self.n) * self.es
        assert np.array_equal(got[:a], self.img[:a]) and np.array_equal(got[b:], self.img[b:]), f"{what}: guard band written"
        return got[a:b].view(NP_BITS[self.kind])


def _eq(got, want, what):
    want = np.ascontiguousarray(want).view(got.dtype)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: {bad.size} of {got.size} elements differ; first at {bad[:8]}"


def _wire_inputs(mode, W, n, rng):
    """Rank buckets of mode `mode` as (bits for the device, oracle input)."""
    xs = [rng.standard_normal(n).astype(np.float32) for _ in range(W)]
    if mode == 2:
        bits = [oracle.f32_to_bf16_bits(x) for x in xs]
        return bits, bits
    if mode == 4:
        bits = [F16.f32_to_f16_bits(x) for x in xs]
        return bits, bits
    return [x.view(np.uint32) for x in xs], xs


def _wire_oracle(mode, inputs, scale):
    return F16.allreduce(mode, inputs, scale) if mode in (3, 4) else oracle.allreduce(mode, inputs, scale)


def _segment_table(spec):
    """spec: [(Buf or None for a zero segment, begin, end)] -> ctypes B2Segment array, built once: only the contents of
    the segments change between replays."""
    segs = (N.B2Segment * len(spec))()
    for k, (b, lo, hi) in enumerate(spec):
        segs[k] = N.B2Segment(N.B2_SEGMENT_ZEROS if b is None else b.t.data_ptr(), lo, hi)
    return segs


class Allreduce:
    def __init__(self, W, mode, algo, n, off=0):
        self.W, self.mode, self.algo, self.n = W, mode, algo, n
        self.bucket, self.wire = WIRE_MODES[mode]
        self.bufs = [Buf(n, self.bucket, off) for _ in range(W)]
        self.what = f"allreduce_ mode={mode} algo={algo} n={n} off={off}"

    def fill(self, rng):
        bits, self.inputs = _wire_inputs(self.mode, self.W, self.n, rng)
        for b, x in zip(self.bufs, bits):
            b.fill(x)

    def launch(self, r, c, s):
        c.allreduce_(self.bufs[r].t, wire=self.wire, algo=self.algo, stream=s)

    def check(self, what):
        want = _wire_oracle(self.mode, self.inputs, 1.0 / self.W)
        for r, b in enumerate(self.bufs):
            _eq(b.read(f"{what} {self.what} rank {r}"), want, f"{what} {self.what} rank {r}")


class Gather:
    """allreduce_gather_ of four segments: an aligned one, a zero segment, a misaligned one and an aligned one."""

    LENS = (1000, 517, 2051, 531)

    def __init__(self, W, mode):
        self.W, self.mode = W, mode
        self.bucket, self.wire = WIRE_MODES[mode]
        self.n = sum(self.LENS)
        self.out = [Buf(self.n, self.bucket, 0) for _ in range(W)]
        self.src = [[Buf(L, self.bucket, off) if k != 1 else None for k, (L, off) in enumerate(zip(self.LENS, (0, 0, 1, 0)))]
                    for _ in range(W)]
        edges = np.cumsum((0,) + self.LENS)
        self.tables = [_segment_table([(b, int(edges[k]), int(edges[k + 1])) for k, b in enumerate(srcs)]) for srcs in self.src]
        self.what = f"allreduce_gather_ mode={mode}"

    def fill(self, rng):
        bits, inputs = _wire_inputs(self.mode, self.W, self.n, rng)
        edges = np.cumsum((0,) + self.LENS)
        self.inputs = []
        for r in range(self.W):
            x = np.array(inputs[r], copy=True)
            for k, b in enumerate(self.src[r]):
                if b is None:
                    x[edges[k]:edges[k + 1]] = 0
                else:
                    b.fill(bits[r][edges[k]:edges[k + 1]])
            self.out[r].fill(np.zeros(self.n, NP_BITS[self.bucket]))
            self.inputs.append(x)

    def launch(self, r, c, s):
        c.allreduce_gather_(self.out[r].t, self.tables[r], len(self.LENS), wire=self.wire, stream=s)

    def check(self, what):
        want = _wire_oracle(self.mode, self.inputs, 1.0 / self.W)
        for r in range(self.W):
            _eq(self.out[r].read(f"{what} {self.what} rank {r}"), want, f"{what} {self.what} rank {r}")
            for b in self.src[r]:
                if b is not None:
                    b.read(f"{what} {self.what} source rank {r}")


class ExactOp:
    """allreduce_op_: int64 sum (wraps), bf16 max, fp32 avg."""

    def __init__(self, W, kind, op, n=3001, off=0):
        self.W, self.kind, self.op, self.n = W, kind, op, n
        self.bufs = [Buf(n, kind, off) for _ in range(W)]
        self.what = f"allreduce_op_ {kind} {op}"

    def fill(self, rng):
        if self.kind == "i64":
            self.inputs = [rng.integers(-2**63, 2**63 - 1, self.n, dtype=np.int64, endpoint=True) for _ in range(self.W)]
        elif self.kind == "bf16":
            self.inputs = [oracle.f32_to_bf16_bits(rng.standard_normal(self.n).astype(np.float32)) for _ in range(self.W)]
        else:
            self.inputs = [rng.standard_normal(self.n).astype(np.float32) for _ in range(self.W)]
        for b, x in zip(self.bufs, self.inputs):
            b.fill(x.view(NP_BITS[self.kind]))

    def launch(self, r, c, s):
        c.allreduce_op_(self.bufs[r].t, self.op, stream=s)

    def check(self, what):
        if self.op == "avg":  # float AVG is the fp32-wire gradient allreduce with scale 1/W
            want = oracle.allreduce(oracle.B2O_F32, self.inputs, 1.0 / self.W) if self.W > 1 else self.inputs[0]
        else:
            want = X.reduce({"i64": "int64", "bf16": "bfloat16"}[self.kind], self.op, self.inputs)
        for r, b in enumerate(self.bufs):
            _eq(b.read(f"{what} {self.what} rank {r}"), want, f"{what} {self.what} rank {r}")


class Allgather:
    def __init__(self, W, n=1027):
        self.W, self.n = W, n
        self.inp = [Buf(n, "u8", 1) for _ in range(W)]
        self.out = [Buf(W * n, "u8", 0) for _ in range(W)]

    def fill(self, rng):
        self.inputs = [rng.integers(0, 256, self.n, dtype=np.uint8) for _ in range(self.W)]
        for r in range(self.W):
            self.inp[r].fill(self.inputs[r])
            self.out[r].fill(np.zeros(self.W * self.n, np.uint8))

    def launch(self, r, c, s):
        c.allgather_(self.out[r].t, self.inp[r].t, stream=s)

    def check(self, what):
        for r in range(self.W):
            _eq(self.out[r].read(f"{what} allgather_ rank {r}"), X.allgather(self.inputs), f"{what} allgather_ rank {r}")


class Broadcast:
    def __init__(self, W, n=5001):
        self.W, self.n, self.root = W, n, W - 1
        self.bufs = [Buf(n, "u8", 3) for _ in range(W)]

    def fill(self, rng):
        self.inputs = [rng.integers(0, 256, self.n, dtype=np.uint8) for _ in range(self.W)]
        for b, x in zip(self.bufs, self.inputs):
            b.fill(x)

    def launch(self, r, c, s):
        c.broadcast_(self.bufs[r].t, root=self.root, stream=s)

    def check(self, what):
        for r, b in enumerate(self.bufs):
            _eq(b.read(f"{what} broadcast_ rank {r}"), self.inputs[self.root], f"{what} broadcast_ root {self.root} rank {r}")


class Reduce:
    """fp32 sum to root 1 % W: the root holds allreduce_op_'s bits, every other rank's buffer is only read."""

    def __init__(self, W, n=4099):
        self.W, self.n, self.root = W, n, 1 % W
        self.bufs = [Buf(n, "f32", 0) for _ in range(W)]

    def fill(self, rng):
        self.inputs = [rng.standard_normal(self.n).astype(np.float32) for _ in range(self.W)]
        for b, x in zip(self.bufs, self.inputs):
            b.fill(x.view(np.uint32))

    def launch(self, r, c, s):
        c.reduce_(self.bufs[r].t, self.root, "sum", stream=s)

    def check(self, what):
        for r, b in enumerate(self.bufs):
            want = oracle.allreduce(oracle.B2O_F32, self.inputs, 1.0) if r == self.root else self.inputs[r]
            _eq(b.read(f"{what} reduce_ rank {r}"), want, f"{what} reduce_ root {self.root} rank {r}")


class ReduceScatter:
    """int32 sum or bf16 avg: block `rank` of the allreduce."""

    def __init__(self, W, kind, op, block=1037):
        self.W, self.kind, self.op, self.block = W, kind, op, block
        self.inp = [Buf(W * block, kind, 0) for _ in range(W)]
        self.out = [Buf(block, kind, 1) for _ in range(W)]
        self.what = f"reduce_scatter_ {kind} {op}"

    def fill(self, rng):
        n = self.W * self.block
        if self.kind == "i32":
            self.inputs = [rng.integers(-2**31, 2**31 - 1, n, dtype=np.int32, endpoint=True) for _ in range(self.W)]
        else:
            self.inputs = [oracle.f32_to_bf16_bits(rng.standard_normal(n).astype(np.float32)) for _ in range(self.W)]
        for r in range(self.W):
            self.inp[r].fill(self.inputs[r])
            self.out[r].fill(np.zeros(self.block, NP_BITS[self.kind]))

    def launch(self, r, c, s):
        c.reduce_scatter_(self.out[r].t, self.inp[r].t, self.op, stream=s)

    def check(self, what):
        if self.kind == "i32":
            full = X.reduce("int32", "sum", self.inputs)
        else:
            full = oracle.allreduce(oracle.B2O_BF16, self.inputs, 1.0 / self.W) if self.W > 1 else self.inputs[0]
        for r in range(self.W):
            _eq(self.out[r].read(f"{what} {self.what} rank {r}"), full[r * self.block:(r + 1) * self.block],
                f"{what} {self.what} rank {r}")
            _eq(self.inp[r].read(f"{what} {self.what} input rank {r}"), self.inputs[r], f"{what} {self.what} input rank {r}")


class ReduceScatterGather:
    """reduce_scatter_gather_ (f32 buckets, bf16 wire) over a padded bucket of W blocks: three segments, the middle one
    zeros, the last one misaligned."""

    def __init__(self, W, block=1555):
        self.W, self.block = W, block
        n = W * block
        self.edges = (0, n // 3, n // 3 + 211, n)
        self.src = [[Buf(self.edges[1], "f32", 0), None, Buf(n - self.edges[2], "f32", 1)] for _ in range(W)]
        self.tables = [_segment_table([(b, self.edges[k], self.edges[k + 1]) for k, b in enumerate(srcs)]) for srcs in self.src]
        self.out = [Buf(block, "f32", 0) for _ in range(W)]

    def fill(self, rng):
        n, e = self.W * self.block, self.edges
        self.inputs = []
        for r in range(self.W):
            x = rng.standard_normal(n).astype(np.float32)
            x[e[1]:e[2]] = 0
            self.src[r][0].fill(x[:e[1]].view(np.uint32))
            self.src[r][2].fill(x[e[2]:].view(np.uint32))
            self.out[r].fill(np.zeros(self.block, np.uint32))
            self.inputs.append(x)

    def launch(self, r, c, s):
        c.reduce_scatter_gather_(self.out[r].t, self.tables[r], 3, wire="bf16", stream=s)

    def check(self, what):
        full = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, self.inputs, 1.0 / self.W)
        for r in range(self.W):
            _eq(self.out[r].read(f"{what} reduce_scatter_gather_ rank {r}"), full[r * self.block:(r + 1) * self.block],
                f"{what} reduce_scatter_gather_ rank {r}")


class Alltoall:
    """Uneven byte splits; every rank sends nothing to the next rank."""

    def __init__(self, W):
        self.W = W
        self.split = [[0 if (W > 1 and j == (i + 1) % W) else (i * 7 + j * 13 + 5) % 41 * 3 + 1 for j in range(W)] for i in range(W)]
        self.ins = [[Buf(self.split[i][j], "u8", (i + j) % 3) for j in range(W)] for i in range(W)]
        self.outs = [[Buf(self.split[j][i], "u8", 1) for j in range(W)] for i in range(W)]

    def fill(self, rng):
        self.data = [[rng.integers(0, 256, self.split[i][j], dtype=np.uint8) for j in range(self.W)] for i in range(self.W)]
        for i in range(self.W):
            for j in range(self.W):
                self.ins[i][j].fill(self.data[i][j])
                self.outs[i][j].fill(np.zeros(self.split[j][i], np.uint8))

    def launch(self, r, c, s):
        c.alltoall_([b.t for b in self.outs[r]], [b.t for b in self.ins[r]], stream=s)

    def check(self, what):
        for i in range(self.W):
            for j in range(self.W):
                _eq(self.outs[i][j].read(f"{what} alltoall_ {j}->{i}"), self.data[j][i], f"{what} alltoall_ {j}->{i}")


class P2pRing:
    """Each rank sends the next one a message of ``nbytes`` and receives the previous rank's.  A message larger than
    ``p2p_eager_bytes`` (all K inbox slots of a channel) reuses slots inside one replay and across replays."""

    def __init__(self, W, nbytes):
        self.W, self.nbytes = W, nbytes
        self.send = [Buf(nbytes, "u8", 0) for _ in range(W)]
        self.recv = [Buf(nbytes, "u8", 1) for _ in range(W)]

    def fill(self, rng):
        self.data = [rng.integers(0, 256, self.nbytes, dtype=np.uint8) for _ in range(self.W)]
        for r in range(self.W):
            self.send[r].fill(self.data[r])
            self.recv[r].fill(np.zeros(self.nbytes, np.uint8))

    def launch(self, r, c, s):
        W = self.W
        c.p2p_([("send", self.send[r].t, (r + 1) % W), ("recv", self.recv[r].t, (r - 1) % W)], stream=s)

    def check(self, what):
        for r in range(self.W):
            _eq(self.recv[r].read(f"{what} p2p_ rank {r}"), self.data[(r - 1) % self.W], f"{what} p2p_ ring into rank {r}")


class BnStats:
    """batchnorm_stats_ with running statistics and counts_out; the last rank has no sample (at W > 1)."""

    def __init__(self, W, C=40, momentum=0.1, eps=1e-5):
        self.W, self.C, self.momentum, self.eps = W, C, momentum, eps
        self.counts = [0.0 if (W > 1 and r == W - 1) else float(3 + 2 * r) for r in range(W)]
        self.b = [{k: Buf(W if k == "counts" else C, "f32", 1 if k in ("invstd", "rv") else 0)
                   for k in ("mean", "invstd", "rm", "rv", "counts")} for _ in range(W)]

    def fill(self, rng):
        W, C = self.W, self.C
        self.means = (rng.standard_normal((W, C)) * 3).astype(np.float32)
        self.invs = rng.uniform(0.2, 5.0, (W, C)).astype(np.float32)
        self.rms = rng.standard_normal((W, C)).astype(np.float32)
        self.rvs = rng.uniform(0.5, 2.0, (W, C)).astype(np.float32)
        for r in range(W):
            for k, v in (("mean", self.means[r]), ("invstd", self.invs[r]), ("rm", self.rms[r]), ("rv", self.rvs[r]),
                         ("counts", np.zeros(W, np.float32))):
                self.b[r][k].fill(v.view(np.uint32))

    def launch(self, r, c, s):
        b = self.b[r]
        c.batchnorm_stats_(b["mean"].t, b["invstd"].t, self.counts[r], b["rm"].t, b["rv"].t, momentum=self.momentum, eps=self.eps,
                           counts_out=b["counts"].t, stream=s)

    def check(self, what):
        mask = torch.tensor(self.counts) >= 1
        dummy = torch.zeros(2, self.C, device="cuda")  # selects ATen's <float, float, int32_t> instance
        for r in range(self.W):
            rm, rv = torch.from_numpy(self.rms[r]).cuda(), torch.from_numpy(self.rvs[r]).cuda()
            wm, wi = torch.batch_norm_gather_stats_with_counts(
                dummy, torch.from_numpy(self.means).cuda()[mask.cuda()], torch.from_numpy(self.invs).cuda()[mask.cuda()], rm, rv,
                self.momentum, self.eps, torch.tensor(self.counts, device="cuda")[mask.cuda()])
            for k, want in (("mean", wm), ("invstd", wi), ("rm", rm), ("rv", rv), ("counts", torch.tensor(self.counts))):
                _eq(self.b[r][k].read(f"{what} batchnorm_stats_ {k} rank {r}"), want.cpu().numpy().astype(np.float32),
                    f"{what} batchnorm_stats_ {k} rank {r}")


class Barrier:
    def fill(self, rng):
        pass

    def launch(self, r, c, s):
        c.barrier(stream=s)

    def check(self, what):
        pass


def _collective_ops(W, multicast, eager_bytes):
    """Graph A's sequence: every collective entry point (p2p only at W > 1)."""
    algos = ["oneshot", "twoshot", "twoshot_ll", "twoshot_pipe"] + (["nvls"] if multicast else [])
    ops = []
    for mode in WIRE_MODES:
        for k, algo in enumerate(algos):
            if algo == "nvls" and mode in (1, 3, 4):
                continue  # NVLS adds on the switch: bf16-wire modes only (its order is not the oracle's, see below)
            ops.append(Allreduce(W, mode, algo, 4099, off=k % 2))
    # buckets larger than a stage region of stage_mb=1: one call, several launches
    ops += [Allreduce(W, 0, "twoshot", 700_000), Allreduce(W, 2, "oneshot", 300_001, off=3),
            Allreduce(W, 4, "twoshot_ll", 600_000, off=1)]
    ops += [Gather(W, 0), Gather(W, 4)]
    ops += [ExactOp(W, "i64", "sum"), ExactOp(W, "bf16", "max", off=1), ExactOp(W, "f32", "avg")]
    ops += [Allgather(W), Broadcast(W), Reduce(W), ReduceScatter(W, "i32", "sum"), ReduceScatter(W, "bf16", "avg"),
            ReduceScatterGather(W), Alltoall(W)]
    if W > 1:
        ops.append(P2pRing(W, eager_bytes + eager_bytes // 8 + 123))  # more than the K inbox slots hold
        assert ops[-1].nbytes > eager_bytes
    ops += [BnStats(W), Barrier()]
    return ops


def _launch_all(world, ops):
    """Eagerly, one op at a time on every rank: the first launch of a kernel (lazy module loading waits for the device)
    never waits behind a collective of rank 0 whose peers have not been issued yet."""
    for op in ops:
        world.run(op.launch)


def _fill_all(ops, seed):
    rng = np.random.default_rng(seed)
    for op in ops:
        op.fill(rng)
    torch.cuda.synchronize()


def _check_all(ops, what):
    for op in ops:
        op.check(what)


@pytest.mark.parametrize("W", [1, 2, 3, 6, 8])
def test_every_collective_replays_against_the_oracle(W):
    world = World([0] * W, stage_mb=1)
    try:
        comms = world.comms
        multicast = comms[0].has_multicast
        eager_bytes = comms[0].p2p_eager_bytes
        ops = _collective_ops(W, multicast, eager_bytes)
        for op in ops:  # NVLS results are checked within the switch's rounding, not bit for bit
            if isinstance(op, Allreduce) and op.algo == "nvls":
                op.check = _nvls_check(op)
        # eager first: loads every kernel, and measures what one pass of the sequence advances the op counter by
        _fill_all(ops, 0)
        before = [c.op_count for c in comms]
        _launch_all(world, ops)
        _check_all(ops, "eager")
        per_graph = comms[0].op_count - before[0]
        if W > 1 and per_graph % 2 == 0:  # an odd count: replay k + 1 starts on the other stage parity from replay k
            ops.append(Barrier())
            _launch_all(world, [ops[-1]])
            per_graph += 1
        assert [c.op_count - b for c, b in zip(comms, before)] == [per_graph] * W
        if W > 1:
            assert per_graph % 2 == 1, per_graph

        # replays cross 2^32 of the op counter
        start = 2**32 - 2 * per_graph - 1
        for c in comms:
            c.set_param("op_count", start)
        launches0 = [c.launches for c in comms]
        graphs = []
        for r, (c, s) in enumerate(zip(comms, world.streams)):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                for op in ops:
                    op.launch(r, c, s)
            graphs.append(g)
        captured = [c.launches - l0 for c, l0 in zip(comms, launches0)]
        assert [c.op_count for c in comms] == [start] * W  # a capture runs nothing
        assert captured[0] > 0

        # Eager work right after the capture and again between replays 2 and 3: it puts the parity and the channel
        # counters out of step with the capture.  Right after the capture, a host-side shadow of the device counters
        # would lead the device by what the capture issued: an LL collective waiting for such a target ends in B2_ETIMEOUT.
        eager = Allreduce(W, 0, "twoshot_ll", 1000, off=1)
        ring = P2pRing(W, eager_bytes // 2 + 5) if W > 1 else None
        eager_ops = 0

        def run_eager(what):
            extra = [eager] + ([ring] if ring else [])
            _fill_all(extra, 7 + eager_ops)
            o0 = comms[0].op_count
            _launch_all(world, extra)
            _check_all(extra, what)
            assert comms[0].op_count - o0 == (1 if W > 1 else 0)
            if W > 1:
                assert [c.last_algo for c in comms] == ["twoshot_ll"] * W
            return comms[0].op_count - o0

        eager_ops += run_eager("eager after the capture")
        for k in range(REPLAYS):
            _fill_all(ops, 100 + k)
            launches, algos = [c.launches for c in comms], [c.last_algo for c in comms]
            world.run(lambda r, c, s: _replay(graphs[r], s))
            _check_all(ops, f"replay {k}")
            # launches and last_algo are host records of the calls that launched: a replay moves neither
            assert [c.launches for c in comms] == launches
            assert [c.last_algo for c in comms] == algos
            if k == 1:
                eager_ops += run_eager("eager between replays")
        assert [c.launches - l0 for c, l0 in zip(comms, launches0)] == [n + (2 * 2 if W > 1 else 2) for n in captured]
        want = (start + per_graph * REPLAYS + eager_ops) % 2**64
        assert [c.op_count for c in comms] == [want] * W
        if W > 1:
            assert want > 2**32 > start
        for c in comms:
            c.check()
    finally:
        world.close()


def _replay(g, s):
    with torch.cuda.stream(s):
        g.replay()


def _nvls_check(op):
    from tests._util import assert_nvls_result

    def check(what):
        for r, b in enumerate(op.bufs):
            got = b.read(f"{what} {op.what} rank {r}")
            got = got.view(np.float32) if op.mode == 0 else got
            assert_nvls_result(got, op.inputs, 1.0 / op.W, op.mode, f"{what} {op.what} rank {r}")

    return check


# ---- Graph B: native BatchNorm2d forward and backward -------------------------------------------------------------
@pytest.mark.parametrize("shape", [(32, 64, 32, 32), (2, 4104, 4, 4)])
def test_native_batchnorm_replays_to_the_bits_of_eager_aten(shape):
    from torchx_b200.nn.bn2d import BatchNorm2d, convert_batchnorm

    n, C, h, w = shape
    if shape[0] == 32:  # the reductions merge over grid_y > 1: their workspace comes from the graph's pool
        geom, nbytes = (ctypes.c_int * 4)(), ctypes.c_size_t()
        N.check(N.lib().b2_bn_reduce_plan(n * h * w, C, geom, ctypes.byref(nbytes)))
        assert geom[3] > 1 and nbytes.value > 0
    torch.manual_seed(3)
    ref = nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        ref.weight.uniform_(0.5, 1.5)
        ref.bias.uniform_(-0.5, 0.5)
    mine = convert_batchnorm(nn.BatchNorm2d(C).cuda())
    mine.load_state_dict(ref.state_dict())
    assert type(mine) is BatchNorm2d
    x = torch.empty(shape, dtype=torch.bfloat16, device="cuda").contiguous(memory_format=torch.channels_last).requires_grad_()
    dy = torch.empty_like(x).requires_grad_(False)

    def fill(seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        with torch.no_grad():
            x.copy_(torch.randn(shape, device="cuda", generator=g) * 2 + 0.5)
            dy.copy_(torch.randn(shape, device="cuda", generator=g))

    def reference():
        xr = x.detach().clone().requires_grad_()
        y = ref(xr)
        saved = (y.grad_fn._saved_result1.clone(), y.grad_fn._saved_result2.clone())
        y.backward(dy)
        out = (y.detach(), xr.grad, ref.weight.grad, ref.bias.grad) + saved
        ref.weight.grad = ref.bias.grad = None
        return out

    fill(1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up, eager, on the side stream: one training step of both
        reference()
        mine(x).backward(dy)
    torch.cuda.synchronize()
    x.grad = mine.weight.grad = mine.bias.grad = None

    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = mine(x)
        saved = y.grad_fn.saved_tensors  # (x, weight, mean, invstd): the graph writes them on every replay
        y.backward(dy)
    outs = [y, x.grad, mine.weight.grad, mine.bias.grad, saved[2], saved[3]]
    names = ["y", "dx", "gw", "gb", "save_mean", "save_invstd"]
    for k in range(4):
        fill(10 + k)
        g.replay()
        torch.cuda.synchronize()
        want = reference()
        for nm, got, wt in zip(names, outs, want):
            assert torch.equal(got.view(torch.int16) if got.dtype == torch.bfloat16 else got.view(torch.int32),
                               wt.view(torch.int16) if wt.dtype == torch.bfloat16 else wt.view(torch.int32)), f"replay {k} {nm}"
        for nm in ("running_mean", "running_var", "num_batches_tracked"):
            assert torch.equal(getattr(mine, nm), getattr(ref, nm)), f"replay {k} {nm}"
    assert int(mine.num_batches_tracked) == 5


# ---- Graph C: a whole mini-DDP training step ------------------------------------------------------------------------
def _net(seed):
    torch.manual_seed(seed)
    m = nn.Sequential(nn.Conv2d(3, 16, 3, padding=1, bias=False), nn.BatchNorm2d(16), nn.ReLU(),
                      nn.Conv2d(16, 32, 3, stride=2, padding=1, bias=False), nn.BatchNorm2d(32), nn.ReLU(),
                      nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(32, 16))
    return m.cuda().to(memory_format=torch.channels_last)


def _batch(r, step):
    g = torch.Generator(device="cuda").manual_seed(1000 * step + r)
    return torch.randn(8, 3, 16, 16, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)


def _loss(ddp, x):
    with torch.autocast("cuda", dtype=torch.bfloat16, cache_enabled=False):  # no cast cache across a capture's edge
        return ddp(x).float().square().mean()


def _step(ddp, opt, x):
    opt.zero_grad(set_to_none=True)
    _loss(ddp, x).backward()
    opt.step()


def _warm_autocast(ddps, streams):
    """tests/test_zero_gpu.py::_warm for this file's convnet under bf16 autocast: a local (no_sync) forward and backward
    per rank loads every compute kernel before any collective is in flight."""
    for r, (d, s) in enumerate(zip(ddps, streams)):
        with torch.cuda.stream(s), d.no_sync():
            _loss(d, _batch(r, 99)).backward()
        d.module.zero_grad(set_to_none=True)
    torch.cuda.synchronize()


def _ddps(W, **kw):
    from tests.test_zero_gpu import _ddps as ddps

    return ddps(W, _net, **kw)


WARMUP, K = 3, 4


@pytest.mark.parametrize("W", [1, 2, 4])
def test_mini_ddp_whole_step_capture_matches_eager_steps(W):
    from tests.test_zero_gpu import _phase

    from torchx_b200.nn.bn2d import BatchNorm2d

    torch.backends.cudnn.deterministic = True
    ca, twin, sa = _ddps(W)
    cb, ddps, sb = _ddps(W)
    try:
        assert any(type(m) is BatchNorm2d for m in ddps[0].module.modules())
        opt_t = [torch.optim.SGD(d.parameters(), lr=0.05, momentum=0.9) for d in twin]
        opt = [torch.optim.SGD(d.parameters(), lr=0.05, momentum=0.9) for d in ddps]
        xs = [_batch(r, 0).clone() for r in range(W)]  # the captured step's static inputs

        def backward(r, step, d, o, s, x=None):
            with torch.cuda.stream(s):
                if x is None:
                    x = _batch(r, step)
                else:
                    x.copy_(_batch(r, step))
                o.zero_grad(set_to_none=True)
                _loss(d, x).backward()

        def opt_step(o, s):
            with torch.cuda.stream(s):
                o.step()

        def eager(step, models, opts, streams, xs=None):
            _phase(W, lambda r: backward(r, step, models[r], opts[r], streams[r], None if xs is None else xs[r]))
            _phase(W, lambda r: opt_step(opts[r], streams[r]))

        _warm_autocast(twin, sa)
        _warm_autocast(ddps, sb)
        # torch's whole-network recipe: warm up on side streams, set the gradients to None, capture on the side stream
        for step in range(WARMUP):
            eager(step, twin, opt_t, sa)
            eager(step, ddps, opt, sb, xs)
        graphs = []
        for r in range(W):
            opt[r].zero_grad(set_to_none=True)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=sb[r]):
                _loss(ddps[r], xs[r]).backward()
                opt[r].step()
            graphs.append(g)
        for k in range(K):
            step = WARMUP + k
            for r in range(W):
                xs[r].copy_(_batch(r, step))
            torch.cuda.synchronize()
            _phase(W, lambda r: _replay(graphs[r], sb[r]))
            for c in cb:  # the forward's health check does not run on a replay
                c.check()
            eager(step, twin, opt_t, sa)
            for r in range(W):
                for (nm, p), q in zip(twin[r].module.named_parameters(), ddps[r].module.parameters()):
                    assert torch.equal(p.view(torch.int32), q.view(torch.int32)), f"replay {k} rank {r} {nm}"
        for r in range(W):
            for p, q in zip(twin[r].module.parameters(), ddps[r].module.parameters()):
                assert torch.equal(opt_t[r].state[p]["momentum_buffer"], opt[r].state[q]["momentum_buffer"])
            for (nm, b), c in zip(twin[r].module.named_buffers(), ddps[r].module.buffers()):
                assert torch.equal(b, c), f"rank {r} {nm}"
    finally:
        for c in ca + cb:
            c.close()


def test_find_unused_parameters_is_refused_under_capture():
    comms, ddps, ss = _ddps(1, find_unused_parameters=True)
    try:
        d, s, c = ddps[0], ss[0], comms[0]
        opt = torch.optim.SGD(d.parameters(), lr=0.05)
        with torch.cuda.stream(s):
            _step(d, opt, _batch(0, 0))
        torch.cuda.synchronize()
        x = _batch(0, 1)
        launches = c.launches
        opt.zero_grad(set_to_none=True)
        with pytest.raises(RuntimeError, match="find_unused_parameters=True cannot run under CUDA graph capture"):
            with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
                _loss(d, x).backward()
        # a backward captured on its own, after an eager forward
        with torch.cuda.stream(s):
            loss = _loss(d, x)
        with pytest.raises(RuntimeError, match="find_unused_parameters=True cannot run under CUDA graph capture"):
            with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
                loss.backward()
        assert c.launches == launches  # refused before any bucket launch
        with torch.cuda.stream(s):  # and the model still trains eagerly
            _step(d, opt, x)
        torch.cuda.synchronize()
        c.check()
    finally:
        for c in comms:
            c.close()


@pytest.mark.parametrize("opt_name", ["adam", "adamw", "sgd"])
def test_zero_overlap_capture_is_refused_or_replays_exactly(opt_name):
    """overlap_with_ddp=True passes step counts and lr by value: a captured step is refused with a RuntimeError.  Should it
    ever be captured, its replays must give the bits of as many eager steps; that is checked first."""
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    cls, kw = {"adam": (torch.optim.Adam, dict(lr=1e-2)), "adamw": (torch.optim.AdamW, dict(lr=1e-2)),
               "sgd": (torch.optim.SGD, dict(lr=0.05, momentum=0.9))}[opt_name]
    torch.backends.cudnn.deterministic = True
    ca, twin, sa = _ddps(1)
    cb, mine, sb = _ddps(1)
    try:
        zt = ZeroRedundancyOptimizer(twin[0], cls, overlap_with_ddp=True, **kw)
        zm = ZeroRedundancyOptimizer(mine[0], cls, overlap_with_ddp=True, **kw)
        x = _batch(0, 0).clone()
        for step in range(2):
            for d, z, s in ((twin[0], zt, sa[0]), (mine[0], zm, sb[0])):
                with torch.cuda.stream(s):
                    x.copy_(_batch(0, step))
                    _step(d, z, x)
                torch.cuda.synchronize()
        zm.zero_grad(set_to_none=True)
        launches = cb[0].launches
        g = torch.cuda.CUDAGraph()
        refused = None
        try:
            with torch.cuda.graph(g, stream=sb[0]):
                _loss(mine[0], x).backward()
                zm.step()
        except RuntimeError as e:
            refused = e
        if refused is None:
            for k in range(3):
                x.copy_(_batch(0, 2 + k))
                torch.cuda.synchronize()
                _replay(g, sb[0])
                with torch.cuda.stream(sa[0]):
                    _step(twin[0], zt, _batch(0, 2 + k))
                torch.cuda.synchronize()
                for (nm, p), q in zip(twin[0].module.named_parameters(), mine[0].module.parameters()):
                    assert torch.equal(p.view(torch.int32), q.view(torch.int32)), f"replay {k} {nm}"
        assert refused is not None and "launch parameters" in str(refused), refused
        assert cb[0].launches == launches  # refused before the first bucket launch
        with torch.cuda.stream(sb[0]):
            with pytest.raises(RuntimeError, match="launch parameters"):
                with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=sb[0]):
                    zm.step()
    finally:
        for c in ca + cb:
            c.close()


# ---- the TMA-staged local pass, first used inside a capture --------------------------------------------------------
_TMA_FIRST_CAPTURE = r"""
import numpy as np
import torch

import oracle
from torchx_b200.ddp import Communicator

(c,) = Communicator.create_local([0], stage_mb=8)
n = 1 << 19  # 2 MiB of fp32, 16-byte aligned: the TMA-staged pass, whose first use sets its shared-memory opt-in
t = torch.empty(n, device="cuda")
s = torch.cuda.Stream()
g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g, stream=s):  # nothing of the library has launched in this process before
    c.allreduce_(t, scale=0.5, wire="bf16", stream=s)
for k in range(3):
    x = np.random.default_rng(k).standard_normal(n).astype(np.float32)
    t.copy_(torch.from_numpy(x))
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        g.replay()
    torch.cuda.synchronize()
    want = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, [x], 0.5)
    assert np.array_equal(t.cpu().numpy().view(np.uint32), want.view(np.uint32)), f"replay {k}"
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    c.allreduce_(t, scale=0.5, wire="bf16")
    torch.cuda.synchronize()
assert any("k_local_pass_tma" in e.name for e in prof.events()), [e.name for e in prof.events()]
c.check()
c.close()
print("ok")
"""


def test_tma_local_pass_first_used_inside_a_capture():
    """At W = 1 a large aligned bucket takes the TMA-staged local pass, whose first launch in a process sets the kernel's
    shared-memory opt-in (cudaFuncSetAttribute).  A fresh process whose first library call is captured must capture that
    launch and replay it to the oracle's bits."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, B2_LOCAL_TMA_MIN_MB="0", PYTHONPATH=root)
    p = subprocess.run([sys.executable, "-c", _TMA_FIRST_CAPTURE], cwd=root, env=env, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and p.stdout.strip().endswith("ok"), p.stdout + p.stderr
