"""Zero segments (B2_SEGMENT_ZEROS) in the gather kernels, against the oracle fed zero-filled arrays for those segments.

The layouts, placements and guard bands are those of tests/test_gather_gpu.py; on top of them some segments of each
rank's table are marked zero: every other one (a vec that crosses from a real segment into a zero one and back), a random
subset, all of them, a head or a tail.  The "ones" layout makes them one element long, "misaligned" puts their neighbours
off a vec.  The result must equal the oracle on the inputs with those segments zeroed, bit for bit (NVLS: its contract),
and the sources must be unchanged.  reduce_scatter_gather_ is checked against the oracle's block, reduce_scatter_step_
against the same step with the zero segments read from real zero tensors."""
import numpy as np
import pytest
import torch

import oracle
from tests._util import MODES, WIRE, World, assert_bits_equal, to_host
from tests.test_gather_gpu import ALGOS, LAYOUTS, PLACEMENTS, _make_ranks, _Solo, _verify
from tests.test_zero_overlap_gpu import HYPER, _table
from torchx_b200.ddp import _native as N
from torchx_b200.ddp import zero as Z

pytestmark = pytest.mark.gpu

PATTERNS = ("alternate", "random", "all", "head", "tail")
DTYPE = {"f32_wire_bf16": torch.float32, "f32": torch.float32, "bf16": torch.bfloat16}


def _zero_segments(pattern, nseg, rng, r):
    if pattern == "alternate":
        return [k for k in range(nseg) if k % 2 == r % 2]
    if pattern == "random":
        return [k for k in range(nseg) if rng.random() < 0.4]
    if pattern == "all":
        return list(range(nseg))
    if pattern == "head":
        return list(range(max(1, nseg // 3)))
    if pattern == "tail":
        return list(range(nseg - max(1, nseg // 3), nseg))
    raise ValueError(pattern)


def _mark_zero(ranks, host, pattern, seed):
    """Marks segments of every rank's table zero and zeroes the oracle's copy of them."""
    rng = np.random.default_rng(seed + 7)
    for r, rk in enumerate(ranks):
        for k in _zero_segments(pattern, len(rk.table), rng, r):
            seg = rk.table[k]
            host[r][seg.begin:seg.end] = 0
            seg.src = N.B2_SEGMENT_ZEROS


def _case(w, n, mode, algo, layout, placement, pattern, seed, kind="randn", out_off=0, stage_mb=8):
    W = len(w.comms)
    scale = 1.0 / W
    ranks, host = _make_ranks([c.device for c in w.comms], n, mode, algo, layout, placement, kind, seed, out_off, stage_mb)
    _mark_zero(ranks, host, pattern, seed)
    w.run(lambda r, c, s: c.allreduce_gather_(ranks[r].out, ranks[r].table, len(ranks[r].table), scale=scale,
                                               wire=WIRE[mode], algo=algo, stream=s))
    what = f"W={W} n={n} mode={mode} algo={algo} layout={layout} placement={placement} zeros={pattern} kind={kind}"
    _verify(ranks, host, mode, scale, w.comms[0].last_algo == "nvls", what)


def _sweep(w, mode, algo, stage_mb=8):
    W = len(w.comms)
    k = 0
    for n in (1, 9, 1023, 8 * 32 * W * 3 - 7, 70001):
        for layout in LAYOUTS if W > 1 else LAYOUTS[:4]:
            pattern = PATTERNS[k % len(PATTERNS)]
            _case(w, n, mode, algo, layout, PLACEMENTS[k % 4], pattern, seed=k, kind=("randn", "special")[k % 2],
                  out_off=(k // 3) % 2, stage_mb=stage_mb)
            k += 1
    for pattern in PATTERNS:  # every pattern on one-element segments and on misaligned neighbours
        _case(w, 1023, mode, algo, "ones", "misaligned", pattern, seed=100 + k, stage_mb=stage_mb)
        _case(w, 4099, mode, algo, "ragged", "mix", pattern, seed=200 + k, kind="nanbits", out_off=1, stage_mb=stage_mb)
        k += 1


@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("algo", ALGOS + ("auto",))
def test_zero_segments_one_device(world, mode, algo):
    w = World([0] * world)
    try:
        _sweep(w, mode, algo)
        if algo == "twoshot_pipe":  # 1 KiB chunks: K > 1 with ragged cells
            for c in w.comms:
                c.set_param("pipe_chunk_bytes", 1 << 10)
            for k, layout in enumerate(("ragged", "ones", "max", "per_rank")):
                _case(w, 8 * 32 * world * 3 - 7, mode, algo, layout, PLACEMENTS[k], PATTERNS[k], seed=300 + k, out_off=k % 2)
    finally:
        w.close()


def test_zero_segments_world1():
    """W = 1: the local pass (k_local_pass) reads the table."""
    w = _Solo()
    try:
        for mode in MODES:
            _sweep(w, mode, "auto")
            _case(w, (1 << 19) + 24, mode, "auto", "max", "misaligned", "random", seed=400)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 4])
def test_zero_segments_chunked_launches(world):
    """stage_mb=1: several launches, each finding its zero segments at bucket coordinate launch offset + element."""
    w = World([0] * world, stage_mb=1)
    try:
        for c in w.comms:
            c.set_param("pipe_chunk_bytes", 32 << 10)
        for i, algo in enumerate(ALGOS):
            _case(w, (3 << 20) + 17, "f32_wire_bf16", algo, "max", PLACEMENTS[i], PATTERNS[i], seed=500 + i, stage_mb=1)
    finally:
        w.close()


def _rs_case(w, block, mode, layout, placement, pattern, seed):
    W = len(w.comms)
    n = W * block
    ranks, host = _make_ranks([c.device for c in w.comms], n, mode, "twoshot", layout, placement, "randn", seed, 0, 8)
    _mark_zero(ranks, host, pattern, seed)
    outs = [torch.full((block,), 7.0, dtype=DTYPE[mode], device="cuda:0") for _ in range(W)]
    w.run(lambda r, c, s: c.reduce_scatter_gather_(outs[r], ranks[r].table, len(ranks[r].table), scale=1.0 / W,
                                                    wire=WIRE[mode], stream=s))
    want = oracle.allreduce(MODES[mode], host, 1.0 / W)
    for r in range(W):
        ranks[r].check_memory(mode, "reduce-scatter sources")
        assert_bits_equal(to_host(outs[r], mode), want[r * block:(r + 1) * block],
                          f"reduce_scatter_gather W={W} block={block} mode={mode} {layout} {placement} zeros={pattern} rank {r}")


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("mode", list(MODES))
def test_zero_segments_reduce_scatter(world, mode):
    w = _Solo() if world == 1 else World([0] * world)
    try:
        k = 0
        for block in (8, 1024, 8 * 1237):
            for layout in ("whole", "ragged", "ones", "max"):
                _rs_case(w, block, mode, layout, PLACEMENTS[k % 4], PATTERNS[k % len(PATTERNS)], seed=600 + k)
                k += 1
    finally:
        w.close()


@pytest.mark.parametrize("kind", ["sgd", "adamw"])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_zero_segments_fused_step(world, kind):
    """The fused step reads a zero segment as the same step does a zero-filled tensor: parameters and state bit-equal."""
    W = world
    w = _Solo() if W == 1 else World([0] * W)
    try:
        sizes = [5, 1, 100, 7, 1000, 3, 64, 2]
        n = sum(sizes)
        B = Z.padded_block(n, W)
        offsets = [sum(sizes[:i]) for i in range(len(sizes))]
        keep, tables = [], {"marker": [], "tensor": []}
        for r in range(W):
            x = torch.randn(n, generator=torch.Generator().manual_seed(700 + r)).cuda()
            zero = torch.zeros(W * B, device="cuda")
            keep += [x, zero]
            for how in tables:
                segs = (N.B2Segment * (len(sizes) + 1))()
                for i, (o, k) in enumerate(zip(offsets, sizes)):
                    unused = (i + r) % 3 == 0
                    src = (N.B2_SEGMENT_ZEROS if how == "marker" else zero.data_ptr()) if unused else x[o:].data_ptr()
                    segs[i].src, segs[i].begin, segs[i].end = src, o, o + k
                segs[len(sizes)].src, segs[len(sizes)].begin, segs[len(sizes)].end = zero.data_ptr(), n, W * B
                tables[how].append(segs)
        gen = torch.Generator().manual_seed(710)
        init = [[torch.randn(B, generator=gen).cuda(), torch.randn(B, generator=gen).cuda(), torch.rand(B, generator=gen).cuda()]
                for _ in range(W)]
        got = {how: [[t.clone() for t in s] for s in init] for how in tables}
        hyper = HYPER[kind][:1]
        for step in range(2):
            for how in tables:
                st = (float(step == 0) if kind == "sgd" else float(step + 1))
                opts = [_table(kind, hyper, B, [(0, 0, st)], *got[how][r]) for r in range(W)]
                w.run(lambda r, c, s: c.reduce_scatter_step_(B, tables[how][r], len(sizes) + 1, opts[r], scale=1.0 / W,
                                                             wire="bf16", stream=s))
        for r in range(W):
            for name, a, b in zip("pmv", got["marker"][r], got["tensor"][r]):
                assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"W={W} {kind} rank {r} {name}"
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("algo", ALGOS + ("nvls", "auto"))
def test_zero_segments_across_devices(world, algo, cuda_count):
    """One rank per device (skipped on a box with fewer GPUs); NVLS reads the table in its cast role."""
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
        for m, mode in enumerate(MODES):
            if algo == "nvls" and mode == "f32":
                continue  # fp32-wire NVLS: the switch's fp32 summation order
            for i, n in enumerate((9, 4099, (1 << 20) + 5)):
                k = 3 * m + i
                _case(w, n, mode, algo, LAYOUTS[k % len(LAYOUTS)], PLACEMENTS[k % 4], PATTERNS[k % len(PATTERNS)], seed=k,
                      kind="special", out_off=k % 2, stage_mb=64)
    finally:
        w.close()
