"""b2_allreduce_gather - the zero-copy bucket fill DistributedDataParallel runs by default - against the oracle.

Each rank's input is read through a segment table (one device pointer per parameter, carried in the kernel parameters)
instead of from the bucket.  Every source allocation and every output bucket carry GUARD elements of POISON on both
sides, and segments sit in separate, guarded slots: a kernel that reads or writes a vec past a segment or bucket boundary
produces a wrong value or a changed guard that the test sees, never an out-of-bounds access.  After each call:
  * the bucket equals the oracle on the concatenation of each rank's segment data (NVLS: the contract of
    tests._util.assert_nvls_result, and the same bits on every rank);
  * every guard element is unchanged;
  * every source that does not alias the bucket is unchanged: the kernels never write their input.
"""
import numpy as np
import pytest
import torch

import oracle
from tests._util import (GUARD, MODES, POISON, WIRE, World, assert_bits_equal, assert_guards_intact, assert_nvls_result,
                         bf16_bits_keep_nan, make_inputs, to_host)
from torchx_b200.ddp import _native as N

pytestmark = pytest.mark.gpu

ALGOS = ("oneshot", "twoshot", "twoshot_pipe", "twoshot_ll")
LAYOUTS = ("whole", "ragged", "ones", "max", "per_rank")
PLACEMENTS = ("mix", "aligned", "misaligned", "alias")
KINDS = ("randn", "special", "nanbits")
RAGGED = (1, 7, 8, 9, 13, 37, 255, 256, 257)
MISALIGN = (1, 3, 4)  # element offsets of a misaligned segment; 4 fp32 = 16 B: aligned for 128-bit, not for a 32 B vec
SLOT = 32             # elements: every segment slot and the bucket start 64 B (bf16) / 128 B (fp32) aligned


def _launches(n, W, mode, algo, stage_mb):
    """[lo, hi) of the launches an explicit algorithm cuts a message of n elements into (a launch holds at most what one
    staging buffer does: one region per rank for one-shot, W regions otherwise)."""
    if W == 1:
        return [(0, n)]
    slice_cap = ((stage_mb << 20) // (W + 1)) & ~255
    cap_vecs = slice_cap // (32 if mode == "f32" else 16)
    max_vecs = cap_vecs if algo == "oneshot" else cap_vecs * W
    out, lo = [], 0
    while lo < n:
        hi = min(n, lo + max_vecs * 8)
        out.append((lo, hi))
        lo = hi
    return out


def _lengths(layout, n, W, launches, rng):
    """Segment lengths of one rank's bucket: at least 1 each, at most B2_MAX_SEGMENTS of them, summing to n."""
    cuts = []
    if layout == "ragged":
        at = 0
        while len(cuts) < N.B2_MAX_SEGMENTS - 1:
            at += RAGGED[len(cuts) % len(RAGGED)]
            if at >= n:
                break
            cuts.append(at)
    elif layout == "ones":  # a 3-element segment, then 40 one-element ones: the vecs [8, 16) .. [32, 40) cross 8 each
        cuts = [c for c in range(3, 44) if c < n]
    elif layout == "max":  # exactly min(n, 128) segments
        want = min(n, N.B2_MAX_SEGMENTS) - 1
        forced = [lo for lo, _ in launches[1:]]  # launch boundaries first, then each launch's slice boundaries and +-1
        for lo, hi in launches:
            Ls = ((hi - lo + 7) // 8 + W - 1) // W
            for j in range(1, W):
                forced += [lo + j * Ls * 8 + d for d in (0, -1, 1)]
        seen = set()
        for c in forced:
            if 0 < c < n and c not in seen and len(seen) < want * 3 // 4:
                seen.add(c)
        while len(seen) < want:
            seen.add(int(rng.integers(1, n)))
        cuts = sorted(seen)
    elif layout != "whole":
        raise ValueError(layout)
    bounds = [0] + cuts + [n]
    return [bounds[i + 1] - bounds[i] for i in range(len(bounds) - 1)]


def _dev(a, device):
    """Host array in the bucket dtype (fp32, or bf16 bits) -> device tensor of that dtype."""
    if a.dtype == np.uint16:
        return torch.from_numpy(a.view(np.int16).copy()).to(f"cuda:{device}").view(torch.bfloat16)
    return torch.from_numpy(a.copy()).to(f"cuda:{device}")


class _Rank:
    """One rank's bucket input `x` cut into segments, the guarded device allocations holding them and the guarded output
    bucket, plus the segment table that points into them."""

    def __init__(self, x, lengths, placements, out_off, device):
        n = x.size
        poison = bf16_bits_keep_nan(np.array([POISON]))[0] if x.dtype == np.uint16 else POISON
        esize = x.itemsize
        begins = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
        starts, pos = [], 0
        for k, pl in enumerate(placements):
            if pl == "alias":
                starts.append(None)
                continue
            pos = -(-(pos + GUARD) // SLOT) * SLOT
            starts.append(pos + (MISALIGN[k % len(MISALIGN)] if pl == "misaligned" else 0))
            pos = starts[-1] + lengths[k]
        self.pool_host = np.full(pos + GUARD, poison, dtype=x.dtype)
        self.lo = SLOT + out_off
        self.hi = self.lo + n
        self.out_host = np.full(self.hi + GUARD, poison, dtype=x.dtype)  # the non-aliased part of the bucket is poisoned
        for k, s in enumerate(starts):
            b, e = begins[k], begins[k + 1]
            if s is None:  # a view of the bucket at its own position, pre-filled with the input
                self.out_host[self.lo + b:self.lo + e] = x[b:e]
            else:
                self.pool_host[s:s + e - b] = x[b:e]
        self.pool = _dev(self.pool_host, device)
        self.out_full = _dev(self.out_host, device)
        self.out = self.out_full[self.lo:self.hi]
        self.table = (N.B2Segment * len(lengths))()
        for k, s in enumerate(starts):
            ptr = self.out_full.data_ptr() + (self.lo + int(begins[k])) * esize if s is None else self.pool.data_ptr() + s * esize
            self.table[k].src, self.table[k].begin, self.table[k].end = ptr, int(begins[k]), int(begins[k + 1])

    def check_memory(self, mode, what):
        """Guards around the bucket intact; every source slot and its guards bit for bit as before.  Returns the bucket."""
        got = to_host(self.out_full, mode)
        assert_guards_intact(got, self.out_host, self.lo, self.hi, f"{what}: bucket guards")
        assert_guards_intact(to_host(self.pool, mode), self.pool_host, 0, 0, f"{what}: sources and their guards")
        return got[self.lo:self.hi]


def _make_ranks(devices, n, mode, algo, layout, placement, kind, seed, out_off, stage_mb):
    W = len(devices)
    rng = np.random.default_rng(seed)
    xs = make_inputs(W, n, seed, kind)
    host = [bf16_bits_keep_nan(x) for x in xs] if mode == "bf16" else xs
    launches = _launches(n, W, mode, algo, stage_mb)
    ranks = []
    for r, d in enumerate(devices):
        lay, pl, off = layout, placement, out_off
        if layout == "per_rank":  # each rank its own table for the same bucket
            lay, pl, off = LAYOUTS[r % 4], PLACEMENTS[(r + r // 4 + seed) % 4], (r + seed) % 2
        lengths = _lengths(lay, n, W, launches, rng)
        places = [PLACEMENTS[1:][i] for i in rng.integers(0, 3, size=len(lengths))] if pl == "mix" else [pl] * len(lengths)
        ranks.append(_Rank(host[r], lengths, places, off, d))
    return ranks, host


def _verify(ranks, host, mode, scale, nvls, what):
    got = [rk.check_memory(mode, f"{what} rank={r}") for r, rk in enumerate(ranks)]
    if nvls:
        for r, g in enumerate(got):
            assert_nvls_result(g, host, scale, MODES[mode], f"{what} rank={r}")
            assert_bits_equal(g, got[0], f"{what}: rank {r} vs rank 0")
        return
    want = oracle.allreduce(MODES[mode], host, scale)
    for r, g in enumerate(got):
        assert_bits_equal(g, want, f"{what} rank={r}")


def _case(w, n, mode, algo, layout, placement, kind, seed, scale=None, out_off=0, stage_mb=8):
    """One gathered allreduce on every rank of `w`, checked."""
    W = len(w.comms)
    scale = 1.0 / W if scale is None else scale
    ranks, host = _make_ranks([c.device for c in w.comms], n, mode, algo, layout, placement, kind, seed, out_off, stage_mb)
    w.run(lambda r, c, s: c.allreduce_gather_(ranks[r].out, ranks[r].table, len(ranks[r].table), scale=scale, wire=WIRE[mode],
                                               algo=algo, stream=s))
    what = (f"W={W} n={n} mode={mode} algo={algo} layout={layout} placement={placement} kind={kind} scale={scale:.4g} "
            f"out_off={out_off} nseg={[len(rk.table) for rk in ranks]}")
    _verify(ranks, host, mode, scale, w.comms[0].last_algo == "nvls", what)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("algo", ALGOS + ("auto",))
def test_gather_matches_oracle_one_device(world, mode, algo):
    w = World([0] * world)
    try:
        sizes = (1, 9, 1023, 8 * 32 * world * 3 - 7, 70001, (1 << 19) + 13)
        for i, n in enumerate(sizes):
            for j, layout in enumerate(LAYOUTS):
                k = i * len(LAYOUTS) + j
                _case(w, n, mode, algo, layout, PLACEMENTS[k % 4], KINDS[k % 3], seed=k, out_off=(k // 3) % 2)
        for k, scale in enumerate((1.0, 1.0 / 3.0)):
            _case(w, 1023, mode, algo, "ragged", "mix", "special", seed=40 + k, scale=scale)
            _case(w, 70001, mode, algo, "max", "misaligned", "nanbits", seed=42 + k, scale=scale, out_off=1)
        if algo == "twoshot_pipe":  # 1 KiB chunks: K > 1 with ragged cells
            for c in w.comms:
                c.set_param("pipe_chunk_bytes", 1 << 10)
            for k, layout in enumerate(("ragged", "ones", "max", "per_rank")):
                _case(w, 8 * 32 * world * 3 - 7, mode, algo, layout, PLACEMENTS[k], KINDS[k % 3], seed=50 + k, out_off=k % 2)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_gather_chunked_launches(world):
    """stage_mb=1: messages are cut into several launches, and each one finds its input at bucket coordinate
    launch offset + element (Src::off)."""
    w = World([0] * world, stage_mb=1)
    try:
        for c in w.comms:
            c.set_param("pipe_chunk_bytes", 32 << 10)
        for i, algo in enumerate(ALGOS):
            before = w.comms[0].launches
            _case(w, (3 << 20) + 17, "f32_wire_bf16", algo, "max", PLACEMENTS[i], KINDS[i % 3], seed=60 + i, out_off=i % 2, stage_mb=1)
            assert w.comms[0].launches - before >= 3, algo
        _case(w, (1 << 20) + 9, "f32", "twoshot", "max", "mix", "randn", seed=64, stage_mb=1)
        _case(w, (1 << 20) + 9, "bf16", "twoshot_ll", "max", "misaligned", "nanbits", seed=65, stage_mb=1)
        _case(w, (1 << 20) + 9, "bf16", "oneshot", "per_rank", "mix", "special", seed=66, stage_mb=1)
    finally:
        w.close()


class _Solo:
    """A one-rank communicator behind the World interface: W = 1 is the fused cast/scale pass over the segments."""

    run = World.run
    close = World.close

    def __init__(self):
        from torchx_b200.ddp import Communicator

        self.comms = [Communicator.create(0, 1, 0, "/unused", stage_mb=8)]
        self.streams = [torch.cuda.current_stream(0)]


def test_gather_world1():
    w = _Solo()
    try:
        for mode in MODES:
            for s, scale in enumerate((1.0, 0.125, 1.0 / 3.0)):
                for j, layout in enumerate(("whole", "ragged", "ones", "max")):
                    k = 4 * s + j
                    _case(w, (1023, 70001, 4099)[k % 3], mode, "auto", layout, PLACEMENTS[k % 4], KINDS[k % 3], seed=k, scale=scale,
                          out_off=k % 2)
            # nothing aliased, the bucket poisoned: F32 at scale 1 must still read the segments (it is no identity here)
            _case(w, 4099, mode, "auto", "ragged", "aligned", "randn", seed=20, scale=1.0)
            # >= 1 MiB and 16 B-aligned: an in-place bucket of this size would stream through the TMA pass, which reads
            # the bucket, not the segments
            _case(w, (1 << 19) + 24, mode, "auto", "max", "misaligned", "special", seed=21, scale=0.125)
            _case(w, (1 << 19) + 24, mode, "auto", "whole", "aligned", "randn", seed=22, scale=1.0)
    finally:
        w.close()


def test_gather_back_to_back_without_sync():
    """30 collectives alternating gather and in-place over mixed algorithms, no host sync in between.  One host table per
    rank is reused and scribbled over right after each call: the call copies it into the kernel parameters."""
    W = 4
    w = World([0] * W)
    try:
        for c in w.comms:
            c.set_param("pipe_chunk_bytes", 1 << 10)
        algos = ("oneshot", "twoshot", "twoshot_pipe", "twoshot_ll", "auto", "twoshot_ll")
        ops = []
        for k in range(30):
            n, algo = 1000 + 53 * k, algos[k % len(algos)]
            if k % 2 == 0:
                lay = LAYOUTS[(k // 2) % len(LAYOUTS)]
                ranks, host = _make_ranks([0] * W, n, "f32_wire_bf16", algo, lay, PLACEMENTS[(k // 2) % 4], KINDS[k % 3], 200 + k,
                                          (k // 2) % 2, 8)
                ops.append((algo, ranks, host))
            else:
                xs = make_inputs(W, n, 200 + k, "randn")
                ops.append((algo, [torch.from_numpy(x).to("cuda:0") for x in xs], xs))
        tables = [(N.B2Segment * N.B2_MAX_SEGMENTS)() for _ in range(W)]
        junk = [torch.full((64,), float(POISON), device="cuda:0") for _ in range(W)]

        def launch(r, c, s):
            tab = tables[r]
            for algo, ranks, _ in ops:
                if isinstance(ranks[r], _Rank):
                    rk = ranks[r]
                    for i, seg in enumerate(rk.table):
                        tab[i].src, tab[i].begin, tab[i].end = seg.src, seg.begin, seg.end
                    c.allreduce_gather_(rk.out, tab, len(rk.table), algo=algo, stream=s)
                    for i in range(len(rk.table)):
                        tab[i].src, tab[i].begin, tab[i].end = junk[r].data_ptr(), 0, 64
                else:
                    c.allreduce_(ranks[r], algo=algo, stream=s)

        w.run(launch)
        for k, (algo, ranks, host) in enumerate(ops):
            what = f"op {k} algo={algo}"
            if isinstance(ranks[0], _Rank):
                _verify(ranks, host, "f32_wire_bf16", 1.0 / W, False, what)
            else:
                want = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, host, 1.0 / W)
                for r in range(W):
                    assert_bits_equal(ranks[r].cpu().numpy(), want, f"{what} rank {r}")
        assert w.comms[0].launches == len(ops)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("algo", ALGOS + ("nvls", "auto"))
def test_gather_across_devices(world, algo, cuda_count):
    """Real NVLink / NVSwitch peers, one rank per device (skipped on a box with fewer GPUs); NVLS reads the segments in its
    cast role and needs the multicast mapping."""
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    w = World(list(range(world)), stage_mb=64)
    try:
        if algo == "nvls" and not w.comms[0].has_multicast:
            pytest.skip("no NVSwitch multicast on this box")
        for c in w.comms:
            c.set_param("pipe_chunk_bytes", 64 << 10)
            c.set_param("nvls_min_bytes", 64 << 10)  # AUTO crosses one-shot -> NVLS / pipelined inside the sizes below
            c.set_param("pipe_min_bytes", 256 << 10)
        for m, mode in enumerate(MODES):
            if algo == "nvls" and mode == "f32":
                continue  # fp32-wire NVLS: the switch's fp32 summation order (tools/nvls_probe.py)
            for i, n in enumerate((9, 4099, (1 << 20) + 5)):
                k = 3 * m + i
                _case(w, n, mode, algo, LAYOUTS[k % len(LAYOUTS)], PLACEMENTS[k % 4], "special", seed=k, out_off=k % 2, stage_mb=64)
            _case(w, (1 << 20) + 5, mode, algo, "max", "mix", "nanbits", seed=10 + m, stage_mb=64)
    finally:
        w.close()
