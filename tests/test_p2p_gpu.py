"""b2_p2p on the GPU: every rank's whole allocation (sent views, received views and the guard bands around them) against a
numpy oracle that matches the k-th receive of every channel with the k-th send, byte for byte; W = 2 .. 8 ranks on one
device.  A ring shift of uint8 / bf16 / fp32 / float64 / int64 at sizes around a vec, a chunk and the eager size and of
64 MiB + 3 bytes, views at every byte offset, several messages on one channel, an asymmetric batch with an idle rank, a
pipeline-shaped batch, an eager send that completes before its receive is launched, 100 rounds interleaved with the
collectives, gather / scatter at every root through the public helpers, the argument checks that need a communicator, a
byte-count mismatch, the public helpers in two processes, and across real devices next to NCCL's batch_isend_irecv at
W = 2 (skipped on a box with fewer GPUs).

Random input bytes make NaNs with every payload in the float dtypes: a copy that went through a float register would show."""
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
from tests._util import World, assert_bits_equal
from tests.test_alltoall_gpu import Exchange, _random_counts
from tests.test_exact_ops_gpu import make_inputs as exact_inputs, to_dev
from torchx_b200.ddp import _native as N

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = {"uint8": torch.uint8, "bfloat16": torch.bfloat16, "float32": torch.float32, "float64": torch.float64,
          "int64": torch.int64}
PAYLOAD = (512 << 10) - 16   # bytes one chunk carries
EAGER = 8 * PAYLOAD          # b2_p2p_eager_bytes
GUARD = 64  # bytes before and after every view, a multiple of 16 so a view's offset mod 16 is the one asked for
STATUS_TEXT = "a point-to-point receive's byte count disagreed with its sender's"


def _esize(dtype):
    return torch.empty(0, dtype=DTYPES[dtype]).element_size()


def _first_diff(got, want):
    bad = np.flatnonzero(got != want)
    return f"{bad.size} bytes differ, first at {bad[:8]}: got {got[bad[:8]]} want {want[bad[:8]]}"


class Batch:
    """One point-to-point batch per rank on a World.  plan[r]: rank r's ops as (kind, peer, bytes, offset), offset = the
    view's byte offset mod 16 (a multiple of the element size); a rank with no ops launches nothing.  Every rank's views live
    in one allocation filled with random bytes, guard bands included."""

    def __init__(self, w, plan, seed, dtype="uint8"):
        self.W, self.plan, self.dtype = len(w.comms), plan, dtype
        rng = np.random.default_rng(seed)
        self.views, self.host = [], []
        for r, c in enumerate(w.comms):
            starts, pos = [], 0
            for _, _, nb, off in plan[r]:
                starts.append(pos + GUARD + off)
                pos = -(-(starts[-1] + nb + GUARD) // 256) * 256
            h = np.frombuffer(rng.bytes(max(pos, 16)), dtype=np.uint8).copy()
            t = torch.from_numpy(h).to(f"cuda:{c.device}")
            self.views.append([t[s:s + nb].view(DTYPES[dtype]) for s, (_, _, nb, _) in zip(starts, plan[r])])
            self.host.append(dict(h=h, t=t, starts=starts))

    def call(self, r, c, s):
        if self.plan[r]:
            c.p2p_([(kind, v, peer) for (kind, peer, _, _), v in zip(self.plan[r], self.views[r])], stream=s)

    def expected(self, r):
        want = self.host[r]["h"].copy()
        for q in range(self.W):
            sends = [i for i, op in enumerate(self.plan[q]) if op[0] == "send" and op[1] == r]
            recvs = [i for i, op in enumerate(self.plan[r]) if op[0] == "recv" and op[1] == q]
            assert len(sends) == len(recvs), f"plan: {len(sends)} sends {q}->{r}, {len(recvs)} receives"
            for i, k in zip(sends, recvs):
                nb = self.plan[r][k][2]
                src = self.host[q]["starts"][i]
                want[self.host[r]["starts"][k]:self.host[r]["starts"][k] + nb] = self.host[q]["h"][src:src + nb]
        return want

    def check(self, ranks=None, what=""):
        for r in range(self.W) if ranks is None else ranks:
            got, want = self.host[r]["t"].cpu().numpy(), self.expected(r)
            assert np.array_equal(got, want), f"{what} W={self.W} {self.dtype} rank {r}: {_first_diff(got, want)}"

    def check_untouched(self, r):
        got = self.host[r]["t"].cpu().numpy()
        assert np.array_equal(got, self.host[r]["h"]), f"rank {r} wrote: {_first_diff(got, self.host[r]['h'])}"


def ring(W, nb, off_send=0, off_recv=0):
    """Send to r + 1, receive from r - 1, in one batch."""
    return [[("send", (r + 1) % W, nb, off_send), ("recv", (r - 1) % W, nb, off_recv)] for r in range(W)]


def test_eager_bytes():
    w = World([0] * 2)
    try:
        assert all(c.p2p_eager_bytes == EAGER == 8 * (512 << 10) - 128 for c in w.comms)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_ring_shift_every_size_and_dtype(world):
    sizes = [0, 1, 15, 16, 17, PAYLOAD, PAYLOAD + 1, EAGER, EAGER + 1]
    w = World([0] * world)
    try:
        for dtype in DTYPES:
            e = _esize(dtype)
            for i, nb in enumerate(sizes):
                x = Batch(w, ring(world, -(-nb // e) * e), seed=i, dtype=dtype)
                before = [c.launches for c in w.comms]
                w.run(x.call)
                x.check(what=f"ring {nb} B")
                assert [c.launches - b for c, b in zip(w.comms, before)] == [1] * world  # one launch per batch
        x = Batch(w, ring(world, (64 << 20) + 3, 5, 11), seed=99)  # 129 chunks per channel: the slots wrap 16 times
        w.run(x.call)
        x.check(what="ring 64 MiB + 3")
    finally:
        w.close()


def test_views_at_every_byte_offset():
    world = 3
    w = World([0] * world)
    try:
        for off in range(16):
            x = Batch(w, ring(world, PAYLOAD + 37 + off, off, (off * 7 + 3) % 16), seed=off)
            w.run(x.call)
            x.check(what=f"offset {off}")
    finally:
        w.close()


def test_several_messages_on_one_channel_arrive_in_order():
    """Rank 0 sends rank 1 six messages in one batch (sizes around a chunk, one empty, one above the eager size) while rank 1
    sends rank 0 three; each receiver lists its receives in the order of its sender's sends, interleaved with its own sends."""
    w = World([0] * 2)
    try:
        a = [17, PAYLOAD + 5, 0, 3, 2 * PAYLOAD, EAGER + 100]
        b = [1000, 1, PAYLOAD - 1]
        plan = [[("send", 1, n, k % 16) for k, n in enumerate(a)] + [("recv", 1, n, 3) for n in b],
                [("recv", 0, n, (5 * k) % 16) for k, n in enumerate(a[:3])] + [("send", 0, n, 1) for n in b]
                + [("recv", 0, n, 0) for n in a[3:]]]
        x = Batch(w, plan, seed=5)
        w.run(x.call)
        x.check()
    finally:
        w.close()


def test_asymmetric_batch_with_an_idle_rank():
    """Only some pairs talk: 0 -> 2 and 2 -> 0 (above the eager size), 1 -> 2 twice; rank 3 launches nothing."""
    w = World([0] * 4)
    try:
        plan = [[("send", 2, EAGER + 7, 0), ("recv", 2, 12345, 1)],
                [("send", 2, 100, 2), ("send", 2, PAYLOAD * 3, 4)],
                [("recv", 1, 100, 5), ("send", 0, 12345, 6), ("recv", 0, EAGER + 7, 7), ("recv", 1, PAYLOAD * 3, 8)],
                []]
        x = Batch(w, plan, seed=6)
        before = w.comms[3].launches
        w.run(x.call)
        x.check()
        assert w.comms[3].launches == before
    finally:
        w.close()


@pytest.mark.parametrize("world", [4, 8])
def test_pipeline_activations_forward_gradients_back(world):
    """Stage r receives activations from r - 1 and gradients from r + 1 and sends its own both ways, in one batch, each
    stage listing its ops in another order."""
    w = World([0] * world)
    try:
        act, grad = 3 * PAYLOAD + 12, EAGER + 2 * PAYLOAD  # bytes: whole fp32 elements
        plan = []
        for r in range(world):
            ops = []
            if r > 0:
                ops += [("recv", r - 1, act, 0), ("send", r - 1, grad, 4)]
            if r < world - 1:
                ops += [("send", r + 1, act, 8), ("recv", r + 1, grad, 12)]
            plan.append(ops[::-1] if r % 2 else ops)
        for dtype in ("bfloat16", "float32"):
            x = Batch(w, plan, seed=world, dtype=dtype)
            w.run(x.call)
            x.check()
    finally:
        w.close()


def test_eager_send_completes_before_its_receive_is_launched():
    """A send of exactly the eager size finishes on its own; only then is the receive launched.  Twice, so the second send
    reuses slots the first receive handed back."""
    w = World([0] * 2)
    try:
        for seed in range(2):
            x = Batch(w, [[("send", 1, EAGER, 3)], [("recv", 0, EAGER, 9)]], seed=seed)
            x.call(0, w.comms[0], w.streams[0])
            w.streams[0].synchronize()
            w.comms[0].check()
            x.call(1, w.comms[1], w.streams[1])
            w.streams[1].synchronize()
            w.comms[1].check()
            x.check()
    finally:
        w.close()


def _random_plan(rng, world):
    """Random pairs, each with 0..3 messages per direction, sizes from empty to above the eager size; at random one idle
    rank.  Each rank shuffles its own list (the order of each channel's messages is kept)."""
    pick = [0, 1, 17, 4096, 100_000, PAYLOAD + 5, 3 * PAYLOAD, EAGER + 9]
    idle = int(rng.integers(world)) if rng.random() < 0.3 else None
    msgs = {}
    for s in range(world):
        for r in range(world):
            if s != r and idle not in (s, r) and rng.random() < 0.5:
                msgs[(s, r)] = [int(rng.choice(pick)) for _ in range(int(rng.integers(1, 4)))]
    plan = [[] for _ in range(world)]
    for (s, r), sizes in msgs.items():
        for n in sizes:
            plan[s].append(("send", r, n, int(rng.integers(16))))
            plan[r].append(("recv", s, n, int(rng.integers(16))))
    for r in range(world):  # interleave channels at random, keeping each channel's own order
        keys = [(op[0], op[1]) for op in plan[r]]
        order = rng.permutation(len(keys))
        queues = {}
        for op in plan[r]:
            queues.setdefault((op[0], op[1]), []).append(op)
        plan[r] = [queues[keys[i]].pop(0) for i in order]
    return plan


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_interleaved_with_the_collectives(world):
    """100 rounds of a random point-to-point batch per rank, then allreduce_op_, allreduce_ and alltoall_ on the same
    communicators, issued back to back, 20 rounds between host syncs: every output against its oracle, bit for bit."""
    w = World([0] * world)
    rounds, n = 100, 3001
    try:
        plan = []
        for k in range(rounds):
            rng = np.random.default_rng(9000 + k)
            ints = exact_inputs("int64", world, 77, seed=k)
            xs = [np.random.default_rng(k * 31 + r).standard_normal(n).astype(np.float32) for r in range(world)]
            plan.append(dict(p=Batch(w, _random_plan(rng, world), seed=k), ints=ints, xs=xs,
                             x=Exchange(w, "int64", _random_counts(rng, world, 8), seed=k),
                             ti=[to_dev(v, "int64", 0) for v in ints], tf=[torch.from_numpy(v.copy()).cuda() for v in xs]))
        torch.cuda.synchronize()

        def ops(r, c, s, p):
            return [lambda: p["p"].call(r, c, s), lambda: c.allreduce_op_(p["ti"][r], "sum", stream=s),
                    lambda: c.allreduce_(p["tf"][r], wire="f32", stream=s), lambda: p["x"].call(r, c, s)]

        # every kernel is loaded first, one synchronised op at a time (tests/test_alltoall_gpu.py says why); round 0's
        # point-to-point batch is re-checked below with the same inputs
        p0 = dict(plan[0], p=Batch(w, plan[0]["p"].plan, seed=0), ti=[t.clone() for t in plan[0]["ti"]],
                  tf=[t.clone() for t in plan[0]["tf"]])
        for o in range(4):
            w.run(lambda r, c, s: ops(r, c, s, p0)[o]())
        for b in range(0, rounds, 20):
            w.run(lambda r, c, s: [op() for p in plan[b:b + 20] for op in ops(r, c, s, p)])
        for k, p in enumerate(plan):
            p["p"].check(what=f"round {k}")
            p["x"].check()
            wi = X.reduce("int64", "sum", p["ints"])
            wf = oracle.allreduce(oracle.B2O_F32, p["xs"], 1.0 / world)
            for r in range(world):
                assert np.array_equal(p["ti"][r].cpu().numpy(), wi), f"round {k} allreduce_op_ rank {r}"
                assert_bits_equal(p["tf"][r].cpu().numpy(), wf, f"round {k} allreduce_ rank {r}")
    finally:
        w.close()


@pytest.mark.parametrize("world", range(1, 9))
def test_gather_and_scatter_every_root(world, monkeypatch):
    """torchx_b200.distributed.gather / scatter on each rank's communicator and stream, every root."""
    import torchx_b200.distributed as D

    w = World([0] * world)
    try:
        def on_rank(fn):
            def call(r, c, s):
                monkeypatch.setattr(D, "_COMM", c)
                with torch.cuda.stream(s):
                    fn(r)
            return call

        n = 1027
        for root in range(world):
            ins = [torch.randint(-2**62, 2**62, (n,), dtype=torch.int64, device="cuda:0") for _ in range(world)]
            lst = [torch.zeros(n, dtype=torch.int64, device="cuda:0") for _ in range(world)]
            torch.cuda.synchronize()
            w.run(on_rank(lambda r: D.gather(ins[r], lst if r == root else None, dst=root)))
            for q in range(world):
                assert torch.equal(lst[q], ins[q]), (root, q)
            chunks = [torch.randint(0, 255, (3 * PAYLOAD + 1,), dtype=torch.uint8, device="cuda:0") for _ in range(world)]
            outs = [torch.zeros(3 * PAYLOAD + 1, dtype=torch.uint8, device="cuda:0") for _ in range(world)]
            torch.cuda.synchronize()
            w.run(on_rank(lambda r: D.scatter(outs[r], chunks if r == root else None, src=root)))
            for q in range(world):
                assert torch.equal(outs[q], chunks[q]), (root, q)
    finally:
        w.close()


def test_argument_validation_with_a_communicator():
    """The checks that need a communicator, through the library: the op count, peers, a null pointer with a count, each
    overlap of a receive; and the contiguity check of p2p_.  Nothing is launched."""
    w = World([0] * 3)
    try:
        L, c = N.lib(), w.comms[1]
        buf = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
        b = buf.data_ptr()

        def call(*ops):
            return L.b2_p2p(c._h, (N.B2P2pOp * len(ops))(*(N.B2P2pOp(*op) for op in ops)), len(ops), None)

        assert L.b2_p2p(c._h, None, 1, None) == N.B2_EINVAL
        assert L.b2_last_error() == b"b2_p2p: null op list"
        for n in (0, 65):
            assert L.b2_p2p(c._h, (N.B2P2pOp * 65)(), n, None) == N.B2_EINVAL
            assert L.b2_last_error() == f"b2_p2p: need 1..64 ops (got {n})".encode()
        for peer in (1, 3, -1):
            assert call((0, 1, b, 16), (peer, 0, b + 64, 16)) == N.B2_EINVAL
            assert L.b2_last_error() == f"b2_p2p: op 1 names peer {peer}; rank 1 of 3 can only name another rank".encode()
        assert call((0, 0, None, 16)) == N.B2_EINVAL
        assert L.b2_last_error() == b"b2_p2p: op 0 has a null pointer and 16 bytes"
        cases = [  # ops as (peer, is_send, ptr, bytes)
            (((0, 0, b, 16), (2, 0, b + 15, 16)), b"op 0 (a recv) overlaps op 1"),
            (((0, 1, b + 100, 8), (2, 0, b, 200)), b"op 1 (a recv) overlaps op 0"),  # a send inside a receive
            (((0, 1, b, 64), (0, 0, b + 63, 1)), b"op 1 (a recv) overlaps op 0"),  # the last byte of a send
            (((0, 0, b, 4), (0, 0, b, 4)), b"op 0 (a recv) overlaps op 1"),
        ]
        for ops, text in cases:
            assert call(*ops) == N.B2_EINVAL, text
            assert text in L.b2_last_error(), (text, L.b2_last_error())
        with pytest.raises(ValueError, match="collectives need a contiguous tensor"):
            c.p2p_([("send", torch.zeros(4, 2, device="cuda:0").t(), 0)])
        assert [cc.launches for cc in w.comms] == [0, 0, 0]
        # what is allowed: sends that overlap each other, an empty range inside another, a null pointer with no bytes.  The
        # batch only sends (eager), so it completes before its peers' receives, queued behind it on the same stream, run.
        assert call((0, 1, b, 64), (2, 1, b, 64), (0, 1, b + 10, 0), (2, 1, None, 0)) == N.B2_OK
        zs = [torch.zeros(64, dtype=torch.uint8, device="cuda:0") for _ in range(3)]
        for r in (0, 2):
            w.comms[r].p2p_([("recv", zs[r], 1), ("recv", zs[r][:0], 1)])
        torch.cuda.synchronize()
        for cc in w.comms:
            cc.check()
        assert all(torch.equal(zs[r], buf[:64]) for r in (0, 2))
        assert [cc.launches for cc in w.comms] == [1, 1, 1]
    finally:
        w.close()


def test_size_mismatch_poisons_only_the_receiver():
    """Rank 2 expects from rank 0 one byte more than rank 0 sends (within the eager size) while ranks 0 and 1 exchange:
    rank 2 writes nothing and reports B2_EINVAL, rank 0's send and everyone else complete normally."""
    w = World([0] * 3, timeout_s=5.0)
    try:
        plan = [[("send", 2, 1000, 0), ("send", 1, 77, 1), ("recv", 1, 5000, 2)],
                [("recv", 0, 77, 3), ("send", 0, 5000, 4)],
                [("recv", 0, 1001, 5)]]
        x = Batch(w, plan, seed=8)
        for r, (c, s) in enumerate(zip(w.comms, w.streams)):
            x.call(r, c, s)
        for s in w.streams:
            s.synchronize()
        x.check([0, 1])
        x.check_untouched(2)
        w.comms[0].check()
        w.comms[1].check()
        with pytest.raises(N.B2Error, match=f"rank 2: {STATUS_TEXT} \\(code -1\\)") as ei:
            w.comms[2].check()
        assert ei.value.code == N.B2_EINVAL
        with pytest.raises(N.B2Error, match=f"communicator poisoned: {STATUS_TEXT}") as ei:
            x.call(2, w.comms[2], w.streams[2])
        assert ei.value.code == N.B2_ESTATE
    finally:
        w.close()


def _run_workers(tmp_path, world, devices, backend, port=0):
    shm = f"/b2_p2p_{uuid.uuid4().hex[:12]}"
    procs = []
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "p2p_worker.py"), "--rank", str(r), "--world",
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
    """Two worker processes on cuda:0 under init_pg("b200") (tests/workers/p2p_worker.py)."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "workers"))
    try:
        import p2p_worker as PW
    finally:
        sys.path.pop(0)
    W = 2
    got = _run_workers(tmp_path, W, [0] * W, "b200")
    for r in range(W):
        for name, want in PW.expected(r, W).items():
            assert got[r][name].dtype == want.dtype and np.array_equal(got[r][name], want), (r, name, got[r][name], want)


@pytest.mark.parametrize("world", [2, 8])
def test_across_devices(world, cuda_count):
    """Real NVLink / NVSwitch peers (skipped on a box with fewer GPUs)."""
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    w = World(list(range(world)), stage_mb=64)
    try:
        for seed in range(3):
            x = Batch(w, _random_plan(np.random.default_rng(seed), world), seed=seed)
            w.run(x.call)
            x.check()
        x = Batch(w, ring(world, (64 << 20) + 3, 5, 11), seed=9)
        w.run(x.call)
        x.check()
    finally:
        w.close()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_equals_nccl_batch_isend_irecv_at_two_gpus(tmp_path, cuda_count):
    """NCCL's batch_isend_irecv and the native batch of the same inputs, bit for bit (one GPU per rank: skipped on a box
    with fewer than two)."""
    if cuda_count < 2:
        pytest.skip("needs 2 GPUs")
    got = _run_workers(tmp_path, 2, [0, 1], "nccl", port=_free_port())
    for r in range(2):
        assert got[r]["nccl_bit_equal"].all(), (r, got[r]["nccl_bit_equal"])
