"""Shared helpers for the parity tests (CPU side: numpy + oracle; GPU side: torch tensors)."""
from __future__ import annotations

import numpy as np

import oracle

# test mode name -> oracle mode, and the wire= argument of Communicator.allreduce_ that selects it
MODES = {"f32_wire_bf16": oracle.B2O_F32_WIRE_BF16, "f32": oracle.B2O_F32, "bf16": oracle.B2O_BF16}
WIRE = {"f32_wire_bf16": "bf16", "f32": "f32", "bf16": "bf16"}

SPECIALS = np.array(
    [0.0, -0.0, np.inf, -np.inf, np.nan, 1e-40, -1e-40, 1.17549435e-38, 3.3895314e38, -3.3895314e38, 1.0, -1.0,
     1.00390625, 1.0078125, 1.01171875, 65504.0, 1e-3, -1e-3, 255.0, 256.0, 257.0],
    dtype=np.float32,
)
# raw fp32 words of the `nanbits` kind: 0xFFFFFFFF is the "not arrived yet" sentinel of the LL / NVLS buffers (and, as
# two bf16 elements 0xFFFF 0xFFFF, the same 32-bit word); quiet NaNs of both signs, a signalling NaN, +-inf
NANBITS = np.array([0xFFFFFFFF, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7F800000, 0xFF800000], dtype=np.uint32)


def make_inputs(world: int, n: int, seed: int, kind: str = "randn") -> list:
    """Per-rank fp32 buckets. kinds: randn (seed 1234+rank as in SURVEY §8d), special (inf/nan/subnormal/
    cancellation sprinkled in), onehot (the reference's own compute_world_size trick), ints (exact in bf16),
    nanbits (randn with the NANBITS words sprinkled in, plus runs of sentinel words so that the bf16 bucket made from it
    by `to_dev` holds 0xFFFF pairs)."""
    out = []
    for r in range(world):
        rng = np.random.default_rng(seed + 1234 + r)
        if kind == "randn":
            x = rng.standard_normal(n).astype(np.float32)
        elif kind == "special":
            x = rng.standard_normal(n).astype(np.float32)
            if n:
                idx = rng.integers(0, n, size=max(1, n // 7))
                x[idx] = SPECIALS[rng.integers(0, len(SPECIALS), size=idx.size)]
                if n > 4:
                    x[1] = 3.25 if r % 2 == 0 else -3.25  # cancellation across rank pairs
        elif kind == "onehot":
            x = np.zeros(n, dtype=np.float32)
            x[r::world] = 1.0
        elif kind == "ints":
            x = rng.integers(-120, 121, size=n).astype(np.float32)
        elif kind == "nanbits":
            x = rng.standard_normal(n).astype(np.float32)
            u = x.view(np.uint32)
            if n:
                idx = rng.integers(0, n, size=max(1, n // 9))
                u[idx] = NANBITS[rng.integers(0, len(NANBITS), size=idx.size)]
                run = rng.integers(0, n, size=max(1, n // 61))
                for k in range(3):  # three consecutive sentinel words: an aligned 0xFFFF pair in bf16 at any offset
                    u[np.minimum(run + k, n - 1)] = 0xFFFFFFFF
        else:
            raise ValueError(kind)
        out.append(x)
    return out


def bf16_bits_keep_nan(x: np.ndarray) -> np.ndarray:
    """bf16 bits of fp32 `x` with round-to-nearest-even, except that a NaN keeps its sign, exponent and the top of its
    payload instead of becoming the canonical NaN, so raw patterns such as 0xFFFF reach a bf16 bucket.  A NaN whose
    payload lives only in the low half (0x7F800001) becomes the signalling bf16 NaN 0x7F81, not an infinity."""
    bits = oracle.f32_to_bf16_bits(x)
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    hi = (u >> 16).astype(np.uint16)
    hi = np.where((hi & 0x7F) == 0, hi | 1, hi).astype(np.uint16)
    bits[nan] = hi[nan]
    return bits


def to_dev(x: np.ndarray, mode: str, device: int):
    """fp32 host data -> (device tensor of the mode's bucket dtype, host copy the oracle takes: fp32 or bf16 bits)."""
    import torch

    if mode == "bf16":
        bits = bf16_bits_keep_nan(x)
        return torch.from_numpy(bits.view(np.int16).copy()).to(f"cuda:{device}").view(torch.bfloat16), bits
    return torch.from_numpy(x.copy()).to(f"cuda:{device}"), x


def to_host(t, mode: str) -> np.ndarray:
    """Device tensor -> fp32 values, or bf16 bits (uint16) for the bf16 mode."""
    import torch

    if mode == "bf16":
        return t.view(torch.int16).cpu().numpy().view(np.uint16)
    return t.cpu().numpy()


class World:
    """`len(devices)` ranks of one communicator inside this process, each launching on its own stream."""

    def __init__(self, devices, stage_mb=8, timeout_s=10.0):
        import torch

        from torchx_b200.ddp import Communicator

        self.comms = Communicator.create_local(devices, stage_mb=stage_mb)
        self.streams = [torch.cuda.Stream(device=d) for d in devices]
        same_device = len(set(devices)) == 1
        for c in self.comms:
            c.set_timeout(timeout_s)
            if same_device:  # all kernels must be co-resident on one GPU: W ranks x grid <= #SMs (1 CTA per SM)
                c.set_max_ctas(max(1, 128 // len(devices)))

    def run(self, fn):
        """fn(rank, comm, stream) launches that rank's work; then wait for all and check health."""
        for r, (c, s) in enumerate(zip(self.comms, self.streams)):
            fn(r, c, s)
        for s in self.streams:
            s.synchronize()
        for c in self.comms:
            c.check()

    def close(self):
        for c in self.comms:
            c.close()


def assert_bits_equal(got: np.ndarray, want: np.ndarray, what: str = "") -> None:
    """Bit-exact comparison; NaNs must coincide but their payload may differ (cvt.rn gives 0x7fff,
    torch's CPU path 0x7fc0)."""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.dtype == np.uint16:
        gf, wf = oracle.bf16_bits_to_f32(got), oracle.bf16_bits_to_f32(want)
        gi, wi = got, want
    else:
        gf, wf = got.astype(np.float32, copy=False), want.astype(np.float32, copy=False)
        gi, wi = gf.view(np.uint32), wf.view(np.uint32)
    gn, wn = np.isnan(gf), np.isnan(wf)
    assert np.array_equal(gn, wn), f"{what}: NaN positions differ at {np.flatnonzero(gn != wn)[:8]}"
    bad = np.flatnonzero((gi != wi) & ~gn)
    assert bad.size == 0, (
        f"{what}: {bad.size} of {got.size} elements differ; first at {bad[:8]}: got {gf[bad[:8]]} want {wf[bad[:8]]}"
    )


GUARD = 16                # elements of guard band on each side of a buffer a kernel is given
POISON = np.float32(1e30)  # what guard bands hold: finite, and far from any value a test reduces


def assert_guards_intact(got: np.ndarray, before: np.ndarray, lo: int, hi: int, what: str = "") -> None:
    """Elements outside [lo, hi) of an allocation are bit for bit what they were before the kernel ran."""
    assert got.dtype == before.dtype and got.shape == before.shape, (what, got.dtype, before.dtype)
    u = np.uint16 if got.dtype == np.uint16 else np.uint32
    gi, bi = got.view(u), before.view(u)
    outside = np.ones(got.size, dtype=bool)
    outside[lo:hi] = False
    bad = np.flatnonzero((gi != bi) & outside)
    assert bad.size == 0, f"{what}: {bad.size} elements outside [{lo}, {hi}) changed; first at {bad[:8]}"


def assert_nvls_result(got: np.ndarray, inputs: list, scale: float, mode: int, what: str = "") -> dict:
    """The NVLS path lets the NVSwitch add the W wire contributions (fp32 accumulation, one rounding to bf16).  The
    switch's summation ORDER is not the rank order of the P2P kernels, so the contract checked here is:
      * wherever the exact sum of the contributions is representable in fp32 along EVERY summation order the result is
        order-independent and must equal the rank-order oracle bit for bit (the overwhelming majority of elements);
      * elsewhere it must equal the correctly rounded bf16 of SOME fp32 summation order: checked as within one bf16 ulp
        of the exact (float64) sum.
    Returns counts for reporting."""
    want = oracle.allreduce(mode, inputs, scale)
    contrib = [oracle.compress(mode, x, scale).astype(np.float64) for x in inputs]  # bf16-representable values
    exact = np.sum(contrib, axis=0)
    if got.dtype == np.uint16:
        gf, wf = oracle.bf16_bits_to_f32(got), oracle.bf16_bits_to_f32(want)
    else:
        gf, wf = got.astype(np.float32), want.astype(np.float32)
    gn, wn = np.isnan(gf), np.isnan(wf)
    assert np.array_equal(gn, wn), f"{what}: NaN positions differ at {np.flatnonzero(gn != wn)[:8]}"
    diff = np.flatnonzero((gf.view(np.uint32) != wf.view(np.uint32)) & ~gn)
    if diff.size:
        # order-independence test: every partial sum of |c_r| spans < 2^24 relative to the smallest contribution bit
        absmax = np.max(np.abs(contrib), axis=0)[diff]
        ulp = np.maximum(np.abs(exact[diff]), np.float64(2.0) ** -126) * 2.0 ** -7  # >= one bf16 ulp of the result
        err = np.abs(gf[diff].astype(np.float64) - exact[diff])
        bad = diff[(err > ulp) & np.isfinite(exact[diff])]
        assert bad.size == 0, (
            f"{what}: {bad.size} elements are more than one bf16 ulp from the exact sum; first at {bad[:8]}: "
            f"got {gf[bad[:8]]} exact {exact[bad[:8]]} rank-order {wf[bad[:8]]}")
        del absmax
    return {"n": int(got.size), "differ_from_rank_order": int(diff.size)}
