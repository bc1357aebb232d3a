"""The fp16 modes on the GPU against tests/oracle_f16.c, bit for bit: B2_F32_WIRE_F16 (fp32 bucket, fp16 wire: the
fp16_compress_hook semantics) and B2_F16 (fp16 bucket).  Every kernel family (local pass plain and TMA, one-shot, two-shot,
pipelined two-shot, LL two-shot, NVLS where the box has multicast), the segment-table gather path, and the DDP front ends
(stock DDP + b200_fp16_compress_hook, the mini-DDP with an fp16 model, with wire="f16" and under GradScaler)."""
import os
import socket
import subprocess
import sys
import uuid

import numpy as np
import pytest
import torch

from tests import _oracle_f16 as F
from tests._util import GUARD, World, assert_guards_intact

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODES = {"f32_wire_f16": F.B2O_F32_WIRE_F16, "f16": F.B2O_F16}
WIRE = "f16"  # the wire= argument; an fp16 bucket is reduced in fp16 whatever it says
POISON32 = np.float32(1e30)
POISON16 = np.uint16(0x5A5A)  # a finite fp16 (203.25), far from anything a test reduces to
SIZES = [1, 7, 8, 9, 1023, 1025, 4099, 32771, (1 << 18) + 5]

# fp16 bit patterns of the `f16bits` kind: the all-ones word half (0xFFFF: a NaN, and as a pair the LL / NVLS sentinel
# word), +-inf, quiet NaNs of both signs, a signalling NaN, the default NaN, the largest finite values, the smallest subnormal
F16BITS = np.array([0xFFFF, 0x7C00, 0xFC00, 0x7E00, 0xFE00, 0x7C01, 0x7FFF, 0x7BFF, 0xFBFF, 0x0001, 0x8001], dtype=np.uint16)
# fp32 words that become such fp16 values (or the fp32 sentinel word itself) in the fp32-bucket mode
F32BITS = np.array([0xFFFFFFFF, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7F800000, 0xFF800000, 0x477FE000, 0x477FF000, 0x33800000],
                   dtype=np.uint32)


def make_inputs(world, n, seed, kind, mode):
    """Per-rank buckets in the bucket's host form: fp32 (f32_wire_f16) or fp16 bits (f16)."""
    out = []
    for r in range(world):
        rng = np.random.default_rng(seed + 4321 + r)
        x = rng.standard_normal(n).astype(np.float32)
        if kind == "special":
            idx = rng.integers(0, n, size=max(1, n // 7))
            x[idx] = rng.choice(np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 65504.0, -65504.0, 65519.0, 65520.0, 1e-7, -3e-8,
                                          6.1e-5, 1.0, 2049.0, 1e5], np.float32), size=idx.size)
        elif kind == "big":  # around 65504 before and after scaling: overflow to inf must survive
            x = (rng.uniform(0.9, 1.1, n) * 65504.0 * rng.choice([1.0, 2.0, 8.0], n) * rng.choice([-1.0, 1.0], n)).astype(np.float32)
        elif kind == "subnormal":  # fp16 subnormal contributions and results
            x = (rng.standard_normal(n) * 2e-6).astype(np.float32)
        elif kind == "ints":
            x = rng.integers(-120, 121, size=n).astype(np.float32)
        elif kind != "randn" and kind != "f16bits":
            raise ValueError(kind)
        if mode == "f16":
            h = F.f32_to_f16_bits(x).copy()
            if kind == "f16bits" and n:
                idx = rng.integers(0, n, size=max(1, n // 9))
                h[idx] = F16BITS[rng.integers(0, len(F16BITS), size=idx.size)]
                run = rng.integers(0, n, size=max(1, n // 61))
                for k in range(3):  # three 0xFFFF in a row: an aligned 0xFFFFFFFF word at any offset
                    h[np.minimum(run + k, n - 1)] = 0xFFFF
            out.append(h)
        else:
            if kind == "f16bits" and n:
                u = x.view(np.uint32)
                idx = rng.integers(0, n, size=max(1, n // 9))
                u[idx] = F32BITS[rng.integers(0, len(F32BITS), size=idx.size)]
            out.append(x)
    return out


def to_dev(h, device=0):
    if h.dtype == np.uint16:
        return torch.from_numpy(h.view(np.int16).copy()).to(f"cuda:{device}").view(torch.float16)
    return torch.from_numpy(h.copy()).to(f"cuda:{device}")


def to_host(t):
    if t.dtype == torch.float16:
        return t.view(torch.int16).cpu().numpy().view(np.uint16)
    return t.cpu().numpy()


def padded(h, lo, hi):
    fill = POISON16 if h.dtype == np.uint16 else POISON32
    return np.concatenate([np.full(lo, fill, h.dtype), h, np.full(hi, fill, h.dtype)])


def _check_allreduce(w, n, mode, algo, kind, seed, offset=0):
    W = len(w.comms)
    xs = make_inputs(W, n, seed, kind, mode)
    full, tens, before = [], [], []
    for r, c in enumerate(w.comms):
        h = padded(xs[r], offset, GUARD)
        t = to_dev(h, c.device)
        full.append(t)
        tens.append(t[offset:offset + n])
        before.append(h)
    scale = 1.0 / W
    w.run(lambda r, c, s: c.allreduce_(tens[r], scale=scale, wire=WIRE, algo=algo, stream=s))
    what = f"W={W} n={n} mode={mode} algo={algo} kind={kind} off={offset}"
    for r in range(W):
        assert_guards_intact(to_host(full[r]), before[r], offset, offset + n, f"{what} rank={r}")
    if w.comms[0].last_algo == "nvls":
        for r in range(W):
            F.assert_nvls_f16_result(to_host(tens[r]), xs, scale, MODES[mode], f"{what} rank={r}")
            F.assert_f16_bits_equal(to_host(tens[r]), to_host(tens[0]), f"{what}: rank {r} vs rank 0")
        return
    want = F.allreduce(MODES[mode], xs, scale)
    for r in range(W):
        F.assert_f16_bits_equal(to_host(tens[r]), want, f"{what} rank={r}")


@pytest.mark.parametrize("mode", list(MODES))
def test_local_pass_matches_oracle(mode):
    """W = 1: the fused cast/scale pass.  The suite's conftest sets B2_LOCAL_TMA_MIN_MB=0 before the library is loaded, so
    every 16 B-aligned bucket of 1 MiB or more takes the TMA-staged kernel, the rest the plain one."""
    from torchx_b200.ddp import local_pass_

    for n in SIZES + [(1 << 19) + 8, (1 << 22) + 3]:
        for kind in ("randn", "special", "f16bits", "big", "subnormal"):
            if kind in ("big", "subnormal", "f16bits") and n > (1 << 19) + 8:
                continue
            for offset in (0, 1):
                h = make_inputs(1, n, 7, kind, mode)[0]
                hp = padded(h, offset, GUARD)
                t = to_dev(hp)
                for scale in (1.0, 0.125, 1.0 / 3.0, 4.0):
                    full = t.clone()
                    tt = full[offset:offset + n]
                    local_pass_(tt, scale=scale, wire=WIRE)
                    torch.cuda.synchronize()
                    what = f"local n={n} mode={mode} kind={kind} scale={scale} off={offset}"
                    assert_guards_intact(to_host(full), hp, offset, offset + n, what)
                    F.assert_f16_bits_equal(to_host(tt), F.allreduce(MODES[mode], [h], scale), what)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("algo", ["oneshot", "twoshot", "twoshot_pipe", "twoshot_ll"])
def test_allreduce_matches_oracle_one_device(world, mode, algo):
    w = World([0] * world)
    try:
        for c in w.comms:
            c.set_param("pipe_chunk_bytes", 16 << 10)
        for i, n in enumerate(SIZES):
            _check_allreduce(w, n, mode, algo, "randn" if i % 2 == 0 else "special", seed=i)
        _check_allreduce(w, 4099, mode, algo, "randn", seed=99, offset=1)  # misaligned base pointer
        _check_allreduce(w, 4099, mode, algo, "f16bits", seed=11)          # NaN payloads, 0xFFFF pairs, +-inf
        _check_allreduce(w, 4099, mode, algo, "f16bits", seed=12, offset=3)
        _check_allreduce(w, 8195, mode, algo, "big", seed=13)              # overflow to inf before / after the scale
        _check_allreduce(w, 8195, mode, algo, "subnormal", seed=14)        # subnormal contributions and results
        _check_allreduce(w, 1 << 12, mode, algo, "ints", seed=0)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_allreduce_auto_and_chunking(world):
    """stage_mb=1: messages cut into several launches, AUTO switching algorithm by size."""
    w = World([0] * world, stage_mb=1)
    try:
        for n in (100, 5000, 70001, (1 << 20) + 17):
            _check_allreduce(w, n, "f32_wire_f16", "auto", "randn", seed=n)
            _check_allreduce(w, n, "f16", "auto", "special", seed=n + 1)
        _check_allreduce(w, (1 << 20) + 11, "f32_wire_f16", "twoshot_ll", "special", seed=7)
        _check_allreduce(w, (1 << 20) + 9, "f16", "twoshot_pipe", "f16bits", seed=8)
    finally:
        w.close()


def _gather_case(w, mode, algo, cuts, misalign, seed):
    """Each rank's bucket input comes from len(cuts) - 1 separate tensors (one per segment), each placed `misalign[k]`
    elements past an aligned allocation start and surrounded by guard elements; the bucket itself only receives the result."""
    from torchx_b200.ddp import _native as N

    W = len(w.comms)
    n = cuts[-1]
    xs = make_inputs(W, n, seed, "f16bits", mode)
    outs, tables, srcs = [], [], []
    for r, c in enumerate(w.comms):
        fill = padded(np.zeros(n, xs[r].dtype), GUARD, GUARD)
        out_full = to_dev(fill, c.device)
        segs = (N.B2Segment * (len(cuts) - 1))()
        mine = []
        for k, (b, e) in enumerate(zip(cuts[:-1], cuts[1:])):
            m = misalign[k % len(misalign)]
            h = padded(xs[r][b:e], GUARD + m, GUARD)
            t = to_dev(h, c.device)
            segs[k].src = t[GUARD + m:].data_ptr()
            segs[k].begin, segs[k].end = b, e
            mine.append((t, h, GUARD + m, GUARD + m + e - b))
        outs.append((out_full, fill))
        tables.append(segs)
        srcs.append(mine)
    w.run(lambda r, c, s: c.allreduce_gather_(outs[r][0][GUARD:GUARD + n], tables[r], len(cuts) - 1, scale=1.0 / W, wire=WIRE,
                                              algo=algo, stream=s))
    want = F.allreduce(MODES[mode], xs, 1.0 / W)
    what = f"gather W={W} mode={mode} algo={algo} segs={len(cuts) - 1}"
    for r in range(W):
        got = to_host(outs[r][0])
        assert_guards_intact(got, outs[r][1], GUARD, GUARD + n, f"{what} rank={r} bucket")
        F.assert_f16_bits_equal(got[GUARD:GUARD + n], want, f"{what} rank={r}")
        for t, h, lo, hi in srcs[r]:  # sources are read only
            assert np.array_equal(to_host(t).view(np.uint8), h.view(np.uint8)), f"{what} rank={r}: a source changed"


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("mode", list(MODES))
def test_segment_table_gather(world, mode):
    w = World([0] * world)
    try:
        ragged = [0, 5, 6, 19, 1000, 1001, 4099, 4107, 9000]  # segments that are not multiples of 8: vecs straddle them
        for algo in (["auto"] if world == 1 else ["oneshot", "twoshot", "twoshot_pipe", "twoshot_ll", "auto"]):
            _gather_case(w, mode, algo, ragged, (0, 1, 3, 4), seed=world)
            _gather_case(w, mode, algo, [0, 70001], (0,), seed=world + 1)
            _gather_case(w, mode, algo, [0, 33, 40000, 70001], (1, 0, 7), seed=world + 2)
    finally:
        w.close()


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("algo", ["twoshot", "twoshot_ll", "nvls", "auto"])
def test_allreduce_across_devices(world, algo, cuda_count):
    """Real NVLink / NVSwitch peers (skipped on a box with fewer GPUs); NVLS against the fp16-ulp contract."""
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    w = World(list(range(world)), stage_mb=64)
    try:
        if algo == "nvls" and not w.comms[0].has_multicast:
            pytest.skip("no NVSwitch multicast on this box")
        for c in w.comms:
            c.set_param("nvls_min_bytes", 64 << 10)
        for mode in MODES:
            for n in (9, 4099, (1 << 20) + 5):
                _check_allreduce(w, n, mode, algo, "special", seed=n)
            _check_allreduce(w, (1 << 20) + 5, mode, algo, "f16bits", seed=3)
            _check_allreduce(w, 1 << 16, mode, algo, "big", seed=4)
    finally:
        w.close()


# ---- DDP front ends: one process per rank (tests/workers/fp16_hook_worker.py) ---------------------------------------------
def _run_workers(world, devices, backend, tmp_path):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    shm = f"/b2_f16_{uuid.uuid4().hex[:12]}"
    procs = []
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "fp16_hook_worker.py"), "--rank", str(r), "--world", str(world),
               "--device", str(devices[r]), "--shm", shm, "--port", str(port), "--backend", backend, "--out", str(tmp_path / f"r{r}.npz")]
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
    got = [dict(np.load(tmp_path / f"r{r}.npz")) for r in range(world)]
    want32 = F.allreduce(F.B2O_F32_WIRE_F16, [g["local"] for g in got], 1.0 / world)
    want16 = F.allreduce(F.B2O_F16, [g["local_half"] for g in got], 1.0 / world)
    for r in range(world):
        F.assert_f16_bits_equal(got[r]["hook"], want32, f"b200_fp16_compress_hook on stock DDP, rank {r}")
        F.assert_f16_bits_equal(got[r]["mini_f16_wire"], want32, f"mini-DDP wire=f16, rank {r}")
        F.assert_f16_bits_equal(got[r]["mini_half"], want16, f"mini-DDP .half() model, rank {r}")
        F.assert_f16_bits_equal(got[r]["hook_half"], want16, f"b200_fp16_compress_hook on a .half() model, rank {r}")
        for k in ("mini_f16_wire_counts", "mini_half_counts"):
            gathered, copied = got[r][k]
            assert gathered > 0 and copied == 0, (k, gathered, copied)  # zero-copy bucket fill throughout
        # GradScaler: rank 0 alone overflowed at step 1; the fp16 wire carried the inf to every rank, so every rank skipped
        # that step and halved its scale, and the parameters stayed identical across ranks
        assert got[r]["scaler_found_inf"].tolist() == [0, 1, 0, 0], got[r]["scaler_found_inf"]
        s = got[r]["scaler_scale"]
        assert s[1] == s[0] / 2 and s[2] == s[1] and s[3] == s[2], s
        assert np.array_equal(got[r]["scaler_params"][1], got[r]["scaler_params"][0])  # step 1 was skipped
        assert not np.array_equal(got[r]["scaler_params"][2], got[r]["scaler_params"][1])  # step 2 was not
        assert np.array_equal(got[r]["scaler_params"].view(np.uint32), got[0]["scaler_params"].view(np.uint32))
    return got


def test_fp16_hook_and_mini_ddp_two_ranks_one_gpu(tmp_path):
    """Both ranks on cuda:0, gloo for stock DDP's bookkeeping."""
    _run_workers(2, [0, 0], "gloo", tmp_path)


@pytest.mark.parametrize("world", [2, 4])
def test_fp16_hook_one_gpu_per_rank_vs_nccl_hook(world, tmp_path, cuda_count):
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    got = _run_workers(world, list(range(world)), "nccl", tmp_path)
    for r in range(world):
        a, b = got[r]["nccl_hook"].astype(np.float64), got[r]["hook"].astype(np.float64)
        if world == 2:  # one fp32 add, one rounding: the reference's fp16_compress_hook over NCCL gives the same bits
            F.assert_f16_bits_equal(got[r]["nccl_hook"], got[r]["hook"], f"NCCL fp16_compress_hook vs ours, rank {r}")
            assert got[r]["nccl_bit_equal"].all(), got[r]["nccl_bit_equal"]
        else:
            assert np.max(np.abs(a - b)) / (np.max(np.abs(b)) + 1e-30) < (world - 1) * 2.0 ** -11
