"""b2_alltoall on the GPU: every rank's outputs against a numpy slicing oracle, byte for byte, with guard bands around every
view; W = 1 .. 8 ranks on one device, uint8 / bf16 / fp32 / float64 / int64, pair sizes around a vec, random uneven split
matrices with an idle rank, views at every byte offset, a pair of exactly the per-pair limit; interleaved with the other
collectives; the argument checks that need a communicator; the over-limit and count-mismatch paths; the
torch.distributed-shaped helpers under init_pg("b200") in two processes; and across real devices, next to NCCL's
all_to_all_single at W = 2 (skipped on a box with fewer GPUs).

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

from tests import _exact_oracle as X
from tests._util import World
from tests.test_exact_ops_gpu import make_inputs as exact_inputs, to_dev
from torchx_b200.ddp import _native as N

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = {"uint8": torch.uint8, "bfloat16": torch.bfloat16, "float32": torch.float32, "float64": torch.float64,
          "int64": torch.int64}
SIZES = [0, 1, 15, 16, 17, (1 << 20) + 3]  # elements per (sender, receiver) pair
GUARD = 64  # bytes before and after every view, a multiple of 16 so a view's offset mod 16 is the one asked for
STATUS_TEXT = "an all-to-all's split sizes disagreed across ranks or exceeded the per-pair limit"


def _esize(dtype):
    return torch.empty(0, dtype=DTYPES[dtype]).element_size()


def _layout(nbytes, offs):
    """Start byte of each view (nbytes[k] bytes at offs[k] past a 256-byte boundary, GUARD bytes around it) and the total."""
    starts, pos = [], 0
    for nb, off in zip(nbytes, offs):
        starts.append(pos + GUARD + off)
        pos = -(-(starts[-1] + nb + GUARD) // 256) * 256
    return starts, pos


def _first_diff(got, want):
    bad = np.flatnonzero(got != want)
    return f"{bad.size} bytes differ, first at {bad[:8]}: got {got[bad[:8]]} want {want[bad[:8]]}"


class Exchange:
    """One all-to-all on a World.  counts[j][r]: elements rank j sends rank r; recv_counts[r][j] (default counts[j][r]):
    elements rank r expects from rank j.  in_offs[j][r] / out_offs[r][j]: byte offset of that view mod 16 (a multiple of
    the element size).  Every buffer is filled with random bytes first, guard bands included."""

    def __init__(self, w, dtype, counts, seed, in_offs=None, out_offs=None, recv_counts=None):
        W = len(w.comms)
        self.W, self.dtype, self.counts = W, dtype, counts
        e = _esize(dtype)
        zero = [[0] * W for _ in range(W)]
        in_offs, out_offs = in_offs or zero, out_offs or zero
        self.recv_counts = recv_counts or [[counts[j][r] for j in range(W)] for r in range(W)]
        rng = np.random.default_rng(seed)
        self.ins, self.outs, self.host = [], [], []
        for r, c in enumerate(w.comms):
            dev = f"cuda:{c.device}"
            si, ni = _layout([counts[r][j] * e for j in range(W)], in_offs[r])
            so, no = _layout([self.recv_counts[r][j] * e for j in range(W)], out_offs[r])
            hi, ho = rng.integers(0, 256, ni, dtype=np.uint8), rng.integers(0, 256, no, dtype=np.uint8)
            ti, to = torch.from_numpy(hi).to(dev), torch.from_numpy(ho).to(dev)
            self.ins.append([ti[s:s + counts[r][j] * e].view(DTYPES[dtype]) for j, s in enumerate(si)])
            self.outs.append([to[s:s + self.recv_counts[r][j] * e].view(DTYPES[dtype]) for j, s in enumerate(so)])
            self.host.append(dict(hi=hi, si=si, ti=ti, ho=ho, so=so, to=to))

    def call(self, r, c, s):
        return c.alltoall_(self.outs[r], self.ins[r], stream=s)

    def what(self, r):
        return f"alltoall W={self.W} {self.dtype} rank={r} counts={self.counts if self.W * self.W <= 16 else '...'}"

    def check(self, ranks=None):
        """Rank r's output allocation holds block r of every rank's input at its views and its old bytes elsewhere."""
        e = _esize(self.dtype)
        for r in range(self.W) if ranks is None else ranks:
            h = self.host[r]
            want = h["ho"].copy()
            for j in range(self.W):
                nb, src = self.counts[j][r] * e, self.host[j]
                want[h["so"][j]:h["so"][j] + nb] = src["hi"][src["si"][r]:src["si"][r] + nb]
            got = h["to"].cpu().numpy()
            assert np.array_equal(got, want), f"{self.what(r)}: {_first_diff(got, want)}"
            assert np.array_equal(h["ti"].cpu().numpy(), h["hi"]), f"{self.what(r)}: the input changed"

    def check_untouched(self, r):
        got = self.host[r]["to"].cpu().numpy()
        assert np.array_equal(got, self.host[r]["ho"]), f"{self.what(r)}: outputs written: {_first_diff(got, self.host[r]['ho'])}"


def launch_all(w, fn):
    """fn(rank, comm, stream) on every rank, then wait; returns {rank: B2Error} of the calls that raised.  No health check."""
    errs = {}
    for r, (c, s) in enumerate(zip(w.comms, w.streams)):
        try:
            fn(r, c, s)
        except N.B2Error as ex:
            errs[r] = ex
    for s in w.streams:
        s.synchronize()
    return errs


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_uniform_pair_sizes_every_dtype(world):
    big = 8 * SIZES[-1]  # bytes of the largest pair (float64)
    w = World([0] * world, stage_mb=8 * (world + 1) + 1)
    try:
        assert w.comms[0].alltoall_max_bytes >= big
        for dtype in DTYPES:
            for i, n in enumerate(SIZES):
                x = Exchange(w, dtype, [[n] * world for _ in range(world)], seed=i)
                before = [c.launches for c in w.comms]
                w.run(x.call)
                x.check()
                assert [c.launches - b for c, b in zip(w.comms, before)] == [int(world > 1)] * world  # one launch, or a copy
    finally:
        w.close()


def _random_counts(rng, world, e, idle=None):
    """A split matrix in elements: zeros, single elements, around a vec, a few KiB and up to ~200 KB per pair."""
    pick = [0, 1, 2, 15, 16, 17, 31, 33, 1000, 4097, 50_001]
    counts = [[int(rng.choice(pick)) for _ in range(world)] for _ in range(world)]
    counts[int(rng.integers(world))][int(rng.integers(world))] = int(rng.integers(1, 200_000 // e))
    if idle is not None:  # sends and receives nothing while the others exchange
        for k in range(world):
            counts[idle][k] = counts[k][idle] = 0
    return counts


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_random_uneven_splits_and_offsets(world):
    w = World([0] * world)
    try:
        for dtype in DTYPES:
            e = _esize(dtype)
            for seed in range(4):
                rng = np.random.default_rng(100 * world + seed)
                counts = _random_counts(rng, world, e, idle=seed % world if seed >= 2 else None)
                offs = [[int(rng.integers(0, 16 // e)) * e for _ in range(world)] for _ in range(2 * world)]
                x = Exchange(w, dtype, counts, seed=seed, in_offs=offs[:world], out_offs=offs[world:])
                w.run(x.call)
                x.check()
    finally:
        w.close()


def test_views_at_every_byte_offset():
    """The send and receive views of uint8 at byte offsets 1..15: every alignment of source, stage and destination."""
    world = 3
    w = World([0] * world)
    try:
        for off in range(1, 16):
            counts = [[37 + 16 * j + r for r in range(world)] for j in range(world)]
            counts[1][2] = 1000 + off
            in_offs = [[off] * world for _ in range(world)]
            out_offs = [[(off * 7 + j) % 16 for j in range(world)] for _ in range(world)]
            x = Exchange(w, "uint8", counts, seed=off, in_offs=in_offs, out_offs=out_offs)
            w.run(x.call)
            x.check()
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 3])
def test_a_pair_of_exactly_the_limit(world):
    w = World([0] * world, stage_mb=1)
    try:
        m = w.comms[0].alltoall_max_bytes
        assert m == (((1 << 20) // (world + 1)) & ~255) - 16 and all(c.alltoall_max_bytes == m for c in w.comms)
        counts = [[5] * world for _ in range(world)]
        counts[0][1], counts[1][0] = m, m - 1
        counts[0][0] = 3 * m  # the own block is copied directly: no limit
        x = Exchange(w, "uint8", counts, seed=1, in_offs=[[3] * world] * world, out_offs=[[9] * world] * world)
        w.run(x.call)
        x.check()
        counts = [[m // 4] * world for _ in range(world)]
        x = Exchange(w, "float32", counts, seed=2)
        w.run(x.call)
        x.check()
    finally:
        w.close()


def test_argument_validation_with_a_communicator():
    """The checks that need a communicator, through the library: a null pointer with a count, each overlap, and (at W = 1)
    the own pair's two counts.  Nothing is launched, so the other rank does not take part."""
    w = World([0] * 2)
    try:
        L, c = N.lib(), w.comms[1]
        buf = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
        b = buf.data_ptr()
        P, S = ctypes.c_void_p * 2, ctypes.c_size_t * 2

        def call(outs, recv, ins, send):
            return L.b2_alltoall(c._h, P(*outs), S(*recv), P(*ins), S(*send), None)

        assert call([None, b + 1024], [16, 16], [b + 2048, b + 3072], [16, 16]) == N.B2_EINVAL
        assert L.b2_last_error() == b"b2_alltoall: out[0] is null but recv_bytes[0] = 16"
        assert call([b, b + 1024], [16, 16], [b + 2048, None], [16, 5]) == N.B2_EINVAL
        assert L.b2_last_error() == b"b2_alltoall: in[1] is null but send_bytes[1] = 5"
        assert L.b2_alltoall(c._h, None, S(1, 1), P(b, b + 16), S(1, 1), None) == N.B2_EINVAL
        assert L.b2_last_error() == b"b2_alltoall: null array"
        assert L.b2_alltoall(c._h, P(b, b + 16), S(1, 1), P(b + 64, b + 80), None, None) == N.B2_EINVAL
        assert L.b2_last_error() == b"b2_alltoall: null array"
        cases = [  # (outs, recv, ins, send, text)
            ([b, b + 15], [16, 16], [b + 1024, b + 2048], [8, 8], b"out[0] overlaps out[1]"),
            ([b + 100, b], [8, 200], [b + 1024, b + 2048], [8, 8], b"out[0] overlaps out[1]"),  # one inside the other
            ([b, b], [4, 4], [b + 1024, b + 2048], [8, 8], b"out[0] overlaps out[1]"),
            ([b, b + 64], [16, 16], [b + 1024, b + 56], [8, 9], b"out[1] overlaps in[1]"),  # the last byte of in[1]
            ([b, b + 64], [16, 16], [b + 15, b + 2048], [8, 8], b"out[0] overlaps in[0]"),
            ([b, b + 64], [16, 16], [b + 2048, b], [8, 16], b"out[0] overlaps in[1]"),  # in place is refused too
        ]
        for outs, recv, ins, send, text in cases:
            assert call(outs, recv, ins, send) == N.B2_EINVAL, text
            assert text in L.b2_last_error(), (text, L.b2_last_error())
        with pytest.raises(ValueError, match="collectives need a contiguous tensor"):
            c.alltoall_([torch.zeros(4, 2, device="cuda:0").t(), buf[:0].float()], [buf[:0].float()] * 2)
        assert w.comms[0].launches == 0 and c.launches == 0
    finally:
        w.close()
    w = World([0])
    try:
        c = w.comms[0]
        x = torch.arange(8, dtype=torch.uint8, device="cuda:0")
        with pytest.raises(N.B2Error, match="rank 0 sends 8 bytes to itself but expects 4") as ei:
            c.alltoall_([torch.zeros(4, dtype=torch.uint8, device="cuda:0")], [x])
        assert ei.value.code == N.B2_EINVAL
        c.check()  # nothing was launched: the communicator is healthy
    finally:
        w.close()


def test_over_limit_pair_gives_up_on_every_rank():
    """One pair of alltoall_max_bytes + 1: its sender's and its receiver's calls raise B2_EINVAL, every rank's kernel gives
    up the exchange without writing an output, and every communicator reports it and refuses further work."""
    world = 3
    w = World([0] * world, stage_mb=1, timeout_s=5.0)
    try:
        m = w.comms[0].alltoall_max_bytes
        counts = [[100] * world for _ in range(world)]
        counts[0][2] = m + 1
        x = Exchange(w, "uint8", counts, seed=3)
        before = [c.launches for c in w.comms]
        errs = launch_all(w, x.call)
        assert sorted(errs) == [0, 2] and all(ex.code == N.B2_EINVAL for ex in errs.values())
        assert f"rank 0 sends {m + 1} bytes to rank 2 and expects 100 from it; one pair carries at most {m}" in str(errs[0])
        assert f"rank 2 sends 100 bytes to rank 0 and expects {m + 1} from it" in str(errs[2])
        assert [c.launches - b for c, b in zip(w.comms, before)] == [1] * world  # the two that raised launched too
        for r, c in enumerate(w.comms):
            x.check_untouched(r)
            with pytest.raises(N.B2Error, match=f"rank {r}: {STATUS_TEXT} \\(code -1\\)") as ei:
                c.check()
            assert ei.value.code == N.B2_EINVAL
        for r, c in enumerate(w.comms):  # poisoned: the argument checks still come first, then the state
            with pytest.raises(N.B2Error, match=f"communicator poisoned: {STATUS_TEXT}") as ei:
                x.call(r, c, w.streams[r])
            assert ei.value.code == N.B2_ESTATE
            with pytest.raises(N.B2Error, match="poisoned"):
                c.allreduce_op_(torch.zeros(4, dtype=torch.int32, device="cuda:0"), "sum")
            with pytest.raises(N.B2Error, match="overlaps"):
                c.alltoall_([x.outs[r][0]] * world, x.ins[r])
    finally:
        w.close()


def test_count_mismatch_poisons_only_the_receiver():
    """Rank 2 expects from rank 0 another count than rank 0 sends, and in a second world rank 1's own two counts differ:
    only that rank writes nothing and reports B2_EINVAL; the others complete with the right bytes."""
    world = 3
    for bad_rank, src, expect in ((2, 0, 41), (1, 1, 7)):
        w = World([0] * world, timeout_s=5.0)
        try:
            counts = [[40 + 10 * j + r for r in range(world)] for j in range(world)]
            recv = [[counts[j][r] for j in range(world)] for r in range(world)]
            recv[bad_rank][src] = expect
            x = Exchange(w, "bfloat16", counts, seed=4, recv_counts=recv)
            assert launch_all(w, x.call) == {}  # only the kernel can see it
            good = [r for r in range(world) if r != bad_rank]
            x.check(good)
            x.check_untouched(bad_rank)
            for r in good:
                w.comms[r].check()
            with pytest.raises(N.B2Error, match=f"rank {bad_rank}: {STATUS_TEXT}") as ei:
                w.comms[bad_rank].check()
            assert ei.value.code == N.B2_EINVAL
        finally:
            w.close()


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_interleaved_with_the_other_collectives(world):
    """100 rounds of alltoall_ (changing dtype, splits and offsets) interleaved with allreduce_op_, allgather_,
    reduce_scatter_ and broadcast_, issued back to back, 20 rounds between host syncs (so that one rank's launch queue
    never fills while the others have issued nothing): every op takes the next stage parity and flag sequence number,
    whatever its kind."""
    w = World([0] * world)
    rounds = 100
    try:
        names = list(DTYPES)
        plan = []
        for k in range(rounds):
            rng = np.random.default_rng(7000 + k)
            dtype = names[k % len(names)]
            e = _esize(dtype)
            counts = _random_counts(rng, world, e, idle=k % world if k % 4 == 0 else None)
            offs = [[int(rng.integers(0, 16 // e)) * e for _ in range(world)] for _ in range(2 * world)]
            ints = exact_inputs("int64", world, 77, seed=k)
            rsi = exact_inputs("int32", world, world * 33, seed=k + 300)
            gat = exact_inputs("int32", world, 19, seed=k + 500)
            bc = [np.full(41, (r + 10 * k) % 256, np.uint8) for r in range(world)]
            plan.append(dict(x=Exchange(w, dtype, counts, seed=k, in_offs=offs[:world], out_offs=offs[world:]), ints=ints,
                             rsi=rsi, gat=gat, bc=bc, root=k % world, op=("sum", "min", "max")[k % 3],
                             ti=[to_dev(v, "int64", 0) for v in ints], trsi=[to_dev(v, "int32", 0) for v in rsi],
                             trsio=[torch.empty(33, dtype=torch.int32, device="cuda:0") for _ in range(world)],
                             tg=[to_dev(v, "int32", 0) for v in gat],
                             tgo=[torch.empty(world * 19, dtype=torch.int32, device="cuda:0") for _ in range(world)],
                             tc=[torch.from_numpy(v.copy()).cuda() for v in bc]))
        torch.cuda.synchronize()

        def ops(r, c, s, p):
            return [lambda: p["x"].call(r, c, s),
                    lambda: c.allreduce_op_(p["ti"][r], p["op"], stream=s),
                    lambda: c.allgather_(p["tgo"][r], p["tg"][r], stream=s),
                    lambda: c.reduce_scatter_(p["trsio"][r], p["trsi"][r], p["op"], stream=s),
                    lambda: c.broadcast_(p["tc"][r], root=p["root"], stream=s)]

        # Every rank is launched from one host thread.  The first launch of a kernel CUDA has not loaded yet waits for the
        # device, i.e. for a collective already spinning on a rank whose launches this thread has not issued, so every
        # kernel of the sequence is loaded first, one synchronised op at a time, on rounds 0-2 (SUM, MIN and MAX).  Their
        # exchanges are re-checked below: the same inputs give the same outputs.
        for p0 in plan[:3]:
            scratch = {k: ([t.clone() for t in v] if k.startswith("t") else v) for k, v in p0.items()}
            for o in range(5):
                w.run(lambda r, c, s: ops(r, c, s, scratch)[o]())

        for b in range(0, rounds, 20):
            w.run(lambda r, c, s: [op() for p in plan[b:b + 20] for op in ops(r, c, s, p)])
        for k, p in enumerate(plan):
            p["x"].check()
            wi = X.reduce("int64", p["op"], p["ints"])
            wrs = X.reduce("int32", p["op"], p["rsi"])
            wg = X.allgather(p["gat"])
            for r in range(world):
                assert np.array_equal(p["ti"][r].cpu().numpy(), wi), f"round {k} allreduce {p['op']} rank {r}"
                assert np.array_equal(p["trsio"][r].cpu().numpy(), wrs[r * 33:(r + 1) * 33]), f"round {k} rs rank {r}"
                assert np.array_equal(p["tgo"][r].cpu().numpy().view(np.uint8), wg), f"round {k} gather rank {r}"
                assert np.array_equal(p["tc"][r].cpu().numpy(), p["bc"][p["root"]]), f"round {k} broadcast rank {r}"
    finally:
        w.close()


def _run_workers(tmp_path, world, devices, backend, port=0):
    shm = f"/b2_a2a_{uuid.uuid4().hex[:12]}"
    procs = []
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "alltoall_worker.py"), "--rank", str(r), "--world",
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
    """Two worker processes on cuda:0 under init_pg("b200") (tests/workers/alltoall_worker.py)."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "workers"))
    try:
        import alltoall_worker as AW
    finally:
        sys.path.pop(0)
    W = 2
    got = _run_workers(tmp_path, W, [0] * W, "b200")
    for r in range(W):
        for name, want in AW.expected(r, W).items():
            assert got[r][name].dtype == want.dtype and np.array_equal(got[r][name], want), (r, name, got[r][name], want)


@pytest.mark.parametrize("world", [2, 8])
def test_across_devices(world, cuda_count):
    """Real NVLink / NVSwitch peers (skipped on a box with fewer GPUs)."""
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    w = World(list(range(world)), stage_mb=64)
    try:
        for dtype in DTYPES:
            e = _esize(dtype)
            for seed in range(3):
                rng = np.random.default_rng(seed)
                counts = _random_counts(rng, world, e, idle=1 if seed == 2 else None)
                x = Exchange(w, dtype, counts, seed=seed, in_offs=[[e * (seed % (16 // e))] * world] * world)
                w.run(x.call)
                x.check()
    finally:
        w.close()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_equals_nccl_all_to_all_single_at_two_gpus(tmp_path, cuda_count):
    """NCCL's all_to_all_single and the native exchange of the same inputs, with and without splits, bit for bit (one GPU
    per rank: skipped on a box with fewer than two)."""
    if cuda_count < 2:
        pytest.skip("needs 2 GPUs")
    got = _run_workers(tmp_path, 2, [0, 1], "nccl", port=_free_port())
    for r in range(2):
        assert got[r]["nccl_bit_equal"].all(), (r, got[r]["nccl_bit_equal"])
