"""Size-independent properties of the oracle's arithmetic (hypothesis), beyond the golden vectors of test_oracle.py:
arbitrary fp32 bit patterns, any world 1..8, any length including ragged tails.  These are the same properties the GPU
parity tests rely on at full bucket sizes (tests/test_allreduce_gpu.py), pinned here on the checker itself."""
import numpy as np
import pytest

hypothesis = pytest.importorskip("hypothesis")
from hypothesis import given, settings  # noqa: E402
from hypothesis import strategies as st  # noqa: E402

import oracle  # noqa: E402
from oracle.ref import allreduce_numpy, bf16_bits_to_f32, f32_to_bf16_bits  # noqa: E402
from tests._util import assert_bits_equal  # noqa: E402

MODES = (oracle.B2O_F32_WIRE_BF16, oracle.B2O_F32)
SETTINGS = dict(max_examples=60, deadline=None)


@st.composite
def buckets(draw, max_world=8, max_n=300, finite_only=False, max_exp=None):
    """Per-rank fp32 buckets made of ARBITRARY bit patterns (NaNs with payloads, infinities, subnormals, both zeros)."""
    world = draw(st.integers(1, max_world))
    n = draw(st.integers(0, max_n))
    seed = draw(st.integers(0, 2 ** 32 - 1))
    rng = np.random.default_rng(seed)
    xs = []
    for _ in range(world):
        bits = rng.integers(0, 2 ** 32, size=n, dtype=np.uint64).astype(np.uint32)
        if finite_only or max_exp is not None:
            lo, hi = (127 - max_exp, 127 + max_exp) if max_exp is not None else (1, 254)
            exp = rng.integers(lo, hi + 1, size=n, dtype=np.uint64).astype(np.uint32)
            bits = (bits & np.uint32(0x807FFFFF)) | (exp << np.uint32(23))
        xs.append(bits.view(np.float32))
    return xs


@settings(**SETTINGS)
@given(buckets(), st.sampled_from([1.0, 0.5, 0.25, 0.125, 1.0 / 3.0, 1.0 / 7.0]))
def test_c_oracle_and_numpy_twin_agree_on_arbitrary_bit_patterns(xs, scale):
    for mode in MODES:
        assert_bits_equal(oracle.allreduce(mode, xs, scale), allreduce_numpy(mode, xs, scale), f"mode {mode} W={len(xs)} n={xs[0].size}")
    xb = [f32_to_bf16_bits(x) for x in xs]
    assert_bits_equal(oracle.allreduce(oracle.B2O_BF16, xb, scale), allreduce_numpy(oracle.B2O_BF16, xb, scale), "bf16 bucket")


@settings(**SETTINGS)
@given(buckets(finite_only=True, max_exp=40), st.integers(-20, 20))
def test_power_of_two_scaling_commutes_with_the_reduction(xs, k):
    """Multiplying every input by 2^k multiplies the result by 2^k exactly (no rounding point moves) as long as nothing
    leaves the normal range - the property that makes the fused 1/W pre-scale safe for W = 2, 4, 8."""
    f = np.float32(2.0 ** k)
    for mode in MODES:
        base = oracle.allreduce(mode, xs, 1.0)
        scaled = oracle.allreduce(mode, [x * f for x in xs], 1.0)
        ok = (np.abs(base) > 1e-25) & (np.abs(base) < 1e25) | (base == 0)  # partial cancellations may dip into subnormals: skip those
        assert_bits_equal(scaled[ok], (base * f)[ok], f"mode {mode}")


@settings(**SETTINGS)
@given(buckets(max_world=2), st.sampled_from([1.0, 0.5]))
def test_two_ranks_commute_and_negation_is_exact(xs, scale):
    if len(xs) == 2:
        for mode in MODES:
            assert_bits_equal(oracle.allreduce(mode, xs, scale), oracle.allreduce(mode, xs[::-1], scale), "a+b == b+a")
    for mode in MODES:  # round-to-nearest-even is symmetric, except for the sign of an exact cancellation (below)
        pos, neg = oracle.allreduce(mode, xs, scale), oracle.allreduce(mode, [-x for x in xs], scale)
        zero = (pos == 0) & (neg == 0)  # c + (-c) is +0 whatever c's sign: both sides may hold +0
        assert_bits_equal(np.where(zero, np.float32(0), neg), np.where(zero, np.float32(0), -pos), "negation")


def test_exact_cancellation_is_positive_zero_on_both_sides():
    """IEEE 754 round-to-nearest: a sum that cancels exactly is +0, and a sum of zeros is -0 only when every zero is -0."""
    a = np.array([1.5, 0.0, -0.0, -0.0, 3e-39], np.float32)
    b = np.array([-1.5, -0.0, 0.0, -0.0, -3e-39], np.float32)
    for mode in MODES:
        for scale in (1.0, 0.5):
            for xs, want in (([a, b], [0, 0, 0, 0x80000000, 0]), ([-a, -b], [0, 0, 0, 0, 0])):
                got = oracle.allreduce(mode, xs, scale)
                assert got.view(np.uint32).tolist() == want, (mode, scale, got.view(np.uint32).tolist())
                assert_bits_equal(got, allreduce_numpy(mode, xs, scale), "numpy twin")


@settings(**SETTINGS)
@given(buckets(), st.sampled_from([1.0, 0.5, 1.0 / 3.0]))
def test_bf16_wire_results_are_bf16_values_and_the_pass_is_idempotent(xs, scale):
    out = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, xs, scale)
    assert_bits_equal(bf16_bits_to_f32(f32_to_bf16_bits(out)), out, "result is bf16-representable")
    # W = 1, scale 1: the local pass (cast, cast back) applied twice equals once - what lets DDP re-reduce a reduced bucket
    once = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, [xs[0]], 1.0)
    assert_bits_equal(oracle.allreduce(oracle.B2O_F32_WIRE_BF16, [once], 1.0), once, "idempotent")
    assert_bits_equal(oracle.compress(oracle.B2O_F32_WIRE_BF16, xs[0], 1.0), once, "compress == W=1 allreduce")


@settings(**SETTINGS)
@given(st.integers(1, 8), st.integers(1, 400), st.integers(0, 2 ** 31))
def test_small_integers_are_summed_exactly_in_any_rank_order(world, n, seed):
    """Integers whose sum stays below 2^8 are exact in bf16 whatever the order - the class of inputs on which ANY correct
    allreduce (NCCL's ring, the switch's tree, our rank order) must agree bit for bit."""
    rng = np.random.default_rng(seed)
    xs = [rng.integers(-15, 16, size=n).astype(np.float32) for _ in range(world)]
    want = np.sum(np.stack(xs), axis=0, dtype=np.float64).astype(np.float32)
    perm = rng.permutation(world)
    for mode in MODES:
        assert_bits_equal(oracle.allreduce(mode, xs, 1.0), want, "exact sum")
        assert_bits_equal(oracle.allreduce(mode, [xs[i] for i in perm], 1.0), want, "any order")


@settings(**SETTINGS)
@given(buckets(max_n=64))
def test_nan_and_infinity_propagate_like_ieee(xs):
    stack = np.stack(xs) if xs[0].size else np.zeros((len(xs), 0), np.float32)
    out = oracle.allreduce(oracle.B2O_F32, xs, 1.0)
    with np.errstate(all="ignore"):
        want_nan = np.isnan(stack).any(axis=0) | (np.isposinf(stack).any(axis=0) & np.isneginf(stack).any(axis=0))
    assert np.all(np.isnan(out)[want_nan])
    with np.errstate(all="ignore"):
        tame = (np.where(np.isfinite(stack), np.abs(stack), 0) < 1e30).all(axis=0)  # finite partial sums cannot overflow to -inf
    only_pos = np.isposinf(stack).any(axis=0) & ~want_nan & tame
    assert np.all(np.isposinf(out[only_pos]))
