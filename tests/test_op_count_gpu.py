"""The flag-synchronised collectives at every op count: a communicator started at a count a long-lived job reaches
(b2_comm_set_param "op_count") must still make every rank wait for every other.

Each collective takes its sequence numbers from the communicator's device op counter, publishes them into flag slots
of its peers and waits until its own slots have caught up: the cta_xbar slot of every CTA index, the pipelined kernels'
slot of every (CTA, kind, chunk) and the LL kernel's flow-control word.  A slot is only rewritten by a launch whose grid
reaches it, so a slot can hold 0 (never written) or a value from any number of operations back when a wider grid, a
larger pipeline or a new kernel comes along.  Such a slot must read as "behind" whatever the count.  Checked here at
counts on both sides of 2^29, 2^30, 2^31 and 2^32 and at 2^40:

* never-written slots: the first collective of a fresh communicator, every entry point, bit for bit against the
  oracles with guard bands;
* aged slots: one op, then the count moved 2^29 + 1 further on, then the same op again;
* no rank finishes alone: rank 0's kernel, launched before any other rank's, must still be running 200 ms later
  (deterministic where the data checks depend on timing);
* the counter itself: k collectives from v leave it at v + k on every rank, and a mixed sequence crosses 2^32 without a
  host sync.

Point-to-point is not tested here: k_p2p never reads the op counter, and the slot of a channel's chunk n is slot n mod 8,
rewritten every 8 chunks of that channel, so its slots cannot go stale."""
import time

import numpy as np
import pytest
import torch

import oracle
from tests import test_allreduce_gpu as AR
from tests import test_alltoall_gpu as A2A
from tests import test_exact_ops_gpu as EO
from tests import test_fp16_gpu as FP
from tests import test_reduce_scatter_gpu as RS
from tests import test_syncbn_gpu as SBN
from tests import test_zero_gpu as ZG
from tests import test_zero_overlap_gpu as ZO
from tests import _exact_oracle as X
from tests._util import World, assert_bits_equal, make_inputs

pytestmark = pytest.mark.gpu

BASES = [0, 2**29 - 3, 2**29, 2**30 - 3, 2**30 + 2**29, 2**31 - 3, 2**32 - 3, 2**40]
WORLDS = [2, 3, 8]
N = 200_003      # allreduce elements: at least 4 CTAs for every algorithm and W here
SOLO_S = 0.2     # how long rank 0's kernel must keep waiting for the others


def _ids(bases):
    return [f"b{b:#x}" for b in bases]


def _world(W, base, max_ctas=None):
    """A fresh communicator of W ranks on cuda:0 (grids capped at 128 / W CTAs, so every rank stays co-resident) whose
    op counter starts at `base`: every flag slot still holds the 0 the arena was created with."""
    w = World([0] * W)
    for c in w.comms:
        c.set_param("op_count", base)
        c.set_param("pipe_chunk_bytes", 16 << 10)  # several pipeline chunks at N
        if max_ctas is not None:
            c.set_max_ctas(max_ctas)
    assert [c.op_count for c in w.comms] == [base] * W  # the knob took: nothing below passes vacuously
    return w


def _counted(w, base, before=0):
    """Every collective launched since the communicator had launched `before` moved every rank's counter by exactly
    one, from `base`."""
    for c in w.comms:
        assert c.op_count == base + c.launches - before, (c.rank, base, c.launches - before, c.op_count)


def _allreduce(mode, algo):
    def case(w):
        if mode == "f32_wire_f16":
            FP._check_allreduce(w, N, mode, algo, "special", seed=3)
        else:
            AR._check_allreduce(w, N, mode, algo, "special", seed=3)
    return case


def _broadcast(w):
    W, nbytes, root = len(w.comms), 100_003, len(w.comms) - 1
    src = np.random.default_rng(5).integers(0, 256, size=nbytes + 1, dtype=np.uint8)
    full = [torch.from_numpy(src.copy() if r == root else np.full(nbytes + 1, r, np.uint8)).cuda() for r in range(W)]
    w.run(lambda r, c, s: c.broadcast_(full[r][:nbytes], root=root, stream=s))
    for r in range(W):
        got = full[r].cpu().numpy()
        assert np.array_equal(got[:nbytes], src[:nbytes]), f"broadcast rank {r}"
        assert got[nbytes] == (src[nbytes] if r == root else r), f"broadcast rank {r}: guard byte"


def _barrier(w):
    w.run(lambda r, c, s: c.barrier(stream=s))


def _alltoall(w):
    W = len(w.comms)
    x = A2A.Exchange(w, "float32", [[30_000 + 7 * (j + r) for r in range(W)] for j in range(W)], seed=9)
    w.run(x.call)
    x.check()


def _bn_stats(w):
    W = len(w.comms)
    SBN.check_stats(w, 2048, [float(3 + 17 * r) for r in range(W)], running=(True, True), momentum=0.1, eps=1e-5, off=1,
                    seed=4)


def _zero(check):
    """check(W), one of the ZeRO tests' checks, on this test's communicator: it takes the communicator from their cache
    (tests/test_zero_gpu._world)."""
    def case(w):
        key = (len(w.comms), 8)
        prev = ZG._WORLDS.get(key)
        ZG._WORLDS[key] = w
        try:
            check(len(w.comms))
        finally:
            if prev is None:
                del ZG._WORLDS[key]
            else:
                ZG._WORLDS[key] = prev
    return case


CASES = {f"allreduce-{mode}-{algo}": _allreduce(mode, algo)
         for mode in ("f32_wire_bf16", "f32", "f32_wire_f16") for algo in ("oneshot", "twoshot", "twoshot_pipe", "twoshot_ll")}
CASES.update({
    "broadcast": _broadcast,
    "barrier": _barrier,
    "allreduce_op": lambda w: EO.check_reduce(w, "int64", "sum", 100_003, seed=1, offset=1),
    "allgather": lambda w: EO.check_gather(w, "int32", 100_003, seed=2, out_off=1),
    "reduce_scatter": lambda w: RS.check_rs(w, "float32", "sum", 100_003, seed=3, out_off=1),
    "alltoall": _alltoall,
    "batchnorm_stats": _bn_stats,
    "reduce_scatter_gather": _zero(lambda W: ZG._check(W, 0, (1 << 17) + 3, seed=6)),
    "reduce_scatter_step": _zero(lambda W: ZO._check(W, 0, (1 << 17) + 3, "sgd0", seed=7, n_steps=1)),  # fused SGD
})


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("base", BASES, ids=_ids(BASES))
@pytest.mark.parametrize("world", WORLDS)
def test_never_written_slots(world, base, case):
    w = _world(world, base)
    try:
        CASES[case](w)
        _counted(w, base)
    finally:
        w.close()


@pytest.mark.parametrize("algo", ["twoshot", "twoshot_pipe"])
@pytest.mark.parametrize("base", BASES, ids=_ids(BASES))
@pytest.mark.parametrize("world", WORLDS)
def test_aged_slots(world, base, algo):
    """Grid 8: slots 0-7 (and, pipelined, their chunk slots) hold this op's sequence numbers; the next op starts 2^29 + 1
    operations later and must not take them for its own."""
    w = _world(world, base, max_ctas=8)
    try:
        AR._check_allreduce(w, 2 * N, "f32_wire_bf16", algo, "randn", seed=1)  # 2N: at least 8 CTAs' worth at every W
        later, before = base + 2**29 + 1, w.comms[0].launches
        for c in w.comms:
            c.set_param("op_count", later)
        AR._check_allreduce(w, 2 * N, "f32_wire_bf16", algo, "special", seed=2)
        _counted(w, later, before)
    finally:
        w.close()


class _RankZeroFirst:
    """A World whose first run() launches rank 0 alone, checks for SOLO_S that its kernel does not complete, and only then
    launches the other ranks; later runs are World's.  The other ranks are launched and every stream synchronised whatever
    happens, so no kernel is left waiting for a rank that never comes."""

    def __init__(self, w):
        self.w, self.comms, self.streams, self.first = w, w.comms, w.streams, True

    def run(self, fn):
        if not self.first:
            return self.w.run(fn)
        self.first = False
        alone = False
        try:
            fn(0, self.comms[0], self.streams[0])
            deadline = time.monotonic() + SOLO_S
            while time.monotonic() < deadline and not alone:
                alone = self.streams[0].query()
                time.sleep(0.002)
        finally:
            for r in range(1, len(self.comms)):
                fn(r, self.comms[r], self.streams[r])
            for s in self.streams:
                s.synchronize()
        assert not alone, "rank 0's collective completed before any other rank had launched"
        for c in self.comms:
            c.check()


# every kernel family that waits on flags, once each; the LL kernel also waits for its peers' data, so it never finishes
# alone even when its flow-control wait is skipped: the data comparisons above are its check
SOLO = ["allreduce-f32_wire_bf16-oneshot", "allreduce-f32_wire_bf16-twoshot", "allreduce-f32_wire_bf16-twoshot_pipe",
        "broadcast", "barrier", "allreduce_op", "allgather", "reduce_scatter", "alltoall", "batchnorm_stats",
        "reduce_scatter_gather", "reduce_scatter_step"]
SOLO_BASES = [2**29 - 3, 2**29, 2**32 - 3]


@pytest.mark.parametrize("case", SOLO)
@pytest.mark.parametrize("base", SOLO_BASES, ids=_ids(SOLO_BASES))
@pytest.mark.parametrize("world", WORLDS)
def test_no_rank_finishes_alone(world, base, case):
    w = _world(world, base)
    try:
        CASES[case](_RankZeroFirst(w))
        _counted(w, base)
    finally:
        w.close()


@pytest.mark.parametrize("world", WORLDS)
def test_interleaved_sequence_crosses_2_32(world):
    """From 2^32 - 5, 12 rounds of bucket allreduce_ (LL, one-shot, two-shot, pipelined in turn), allreduce_op_,
    allgather_ and broadcast_, issued back to back without a host sync: the count passes 2^32 in the second round with
    the stage parity still alternating, every result matches its oracle and the counter ends 48 operations on."""
    w = World([0] * world)
    rounds, n = 12, 5000
    algos = ("twoshot_ll", "oneshot", "twoshot", "twoshot_pipe")
    try:
        for c in w.comms:
            c.set_param("pipe_chunk_bytes", 1 << 10)
        plan = []
        for k in range(rounds):
            b = make_inputs(world, n, 100 + k, "special")
            ints = EO.make_inputs("int64", world, 999, seed=k)
            gat = EO.make_inputs("int32", world, 37, seed=k + 500)
            bc = [np.full(4099, (r + 10 * k) % 256, np.uint8) for r in range(world)]
            plan.append(dict(b=b, ints=ints, gat=gat, bc=bc, root=k % world, op=("sum", "min", "max")[k % 3],
                             algo=algos[k % 4],
                             tb=[torch.from_numpy(x.copy()).cuda() for x in b],
                             ti=[EO.to_dev(x, "int64", 0) for x in ints],
                             tg=[EO.to_dev(x, "int32", 0) for x in gat],
                             tgo=[torch.empty(world * 37, dtype=torch.int32, device="cuda:0") for _ in range(world)],
                             tc=[torch.from_numpy(x.copy()).cuda() for x in bc]))
        torch.cuda.synchronize()

        def ops(r, c, s, p):
            return [lambda: c.allreduce_(p["tb"][r], wire="bf16", algo=p["algo"], stream=s),
                    lambda: c.allreduce_op_(p["ti"][r], p["op"], stream=s),
                    lambda: c.allgather_(p["tgo"][r], p["tg"][r], stream=s),
                    lambda: c.broadcast_(p["tc"][r], root=p["root"], stream=s)]

        # Every kernel of the sequence is loaded first, one synchronised op at a time, on scratch copies of rounds 0-3
        # (a kernel's first launch waits for the device, i.e. for a rank already spinning on ranks not launched yet).
        for p0 in plan[:4]:
            scratch = {k: ([t.clone() for t in v] if k.startswith("t") else v) for k, v in p0.items()}
            for o in range(4):
                w.run(lambda r, c, s: ops(r, c, s, scratch)[o]())
        base = 2**32 - 5
        for c in w.comms:
            c.set_param("op_count", base)
        w.run(lambda r, c, s: [op() for p in plan for op in ops(r, c, s, p)])
        for k, p in enumerate(plan):
            wb = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, p["b"], 1.0 / world)
            wi = X.reduce("int64", p["op"], p["ints"])
            wg = X.allgather(p["gat"])
            for r in range(world):
                assert_bits_equal(p["tb"][r].cpu().numpy(), wb, f"round {k} {p['algo']} rank {r}")
                assert np.array_equal(EO.to_host(p["ti"][r], "int64"), wi), f"round {k} {p['op']} rank {r}"
                assert np.array_equal(EO.to_host(p["tgo"][r], "int32").view(np.uint8), wg), f"round {k} gather rank {r}"
                assert np.array_equal(p["tc"][r].cpu().numpy(), p["bc"][p["root"]]), f"round {k} broadcast rank {r}"
        assert [c.op_count for c in w.comms] == [base + 4 * rounds] * world
    finally:
        w.close()
