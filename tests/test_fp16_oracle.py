"""The fp16 modes (B2_F32_WIRE_F16 = 3, B2_F16 = 4) without a GPU: the C oracle's binary16 rounding against numpy's and
torch's, the oracle against the reference's own DDP runs (tests/golden/ddp_fp16_w{2,4}.npz), the header against the
binding, the AUTO policy table, and the dtype / wire -> mode mapping."""
import os
import re

import numpy as np
import pytest
import torch

from tests import _oracle_f16 as F
from torchx_b200.ddp import _native as N
from torchx_b200.ddp.comm import mode_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MIB = 1 << 20

# the targeted rounding cases: the largest finite values, the overflow tie, the subnormal range and its ties, signed zero
TARGETED = np.array(
    [65504.0, 65519.0, 65519.996, 65520.0, -65520.0, 65536.0, 1e9, -1e9, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25,
     -(2.0 ** -25), 2.0 ** -26, 5 * 2.0 ** -26, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -25, 2.0 ** -14 - 2.0 ** -24, 6.1e-5,
     1.0, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -20, 2049.0, 2051.0, -0.0, 0.0, 1e-45, -1e-40,
     np.inf, -np.inf, 0.1, -0.3, 3.14159265],
    dtype=np.float32,
)
NAN_WORDS = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x7FBFFFFF], dtype=np.uint32)


def _torch_f16_bits(x: np.ndarray) -> np.ndarray:
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.float16).view(torch.int16).numpy().view(np.uint16)


def _check_rne(x: np.ndarray) -> None:
    c, npy, tor = F.f16_rne(x), F.f32_to_f16_bits(x), _torch_f16_bits(x)
    nan = np.isnan(x)
    # NaNs: every conversion must give a NaN (payloads differ: the oracle gives the cvt.rn default NaN 0x7fff)
    for name, b in (("oracle", c), ("numpy", npy), ("torch", tor)):
        assert np.all(np.isnan(F.f16_bits_to_f32(b[nan]))), name
    assert np.array_equal(c[~nan], npy[~nan]), x[~nan][c[~nan] != npy[~nan]][:8]
    assert np.array_equal(c[~nan], tor[~nan]), x[~nan][c[~nan] != tor[~nan]][:8]


def test_f16_rounding_targeted_cases():
    _check_rne(np.concatenate([TARGETED, NAN_WORDS.view(np.float32)]))
    b = F.f16_rne(np.array([65504.0, 65519.0, 65520.0, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25, -0.0], np.float32))
    assert b.tolist() == [0x7BFF, 0x7BFF, 0x7C00, 0x0001, 0x0000, 0x0002, 0x8000]


def test_f16_rounding_random_bit_patterns():
    rng = np.random.default_rng(5)
    words = rng.integers(0, 1 << 32, size=40_000, dtype=np.uint64).astype(np.uint32)
    # and a dense sweep of the fp16 range, where the interesting roundings happen (subnormals, normals, overflow)
    exps = rng.integers(100, 145, size=40_000).astype(np.uint32)
    near = (exps << 23) | rng.integers(0, 1 << 23, size=40_000).astype(np.uint32) | (rng.integers(0, 2, size=40_000).astype(np.uint32) << 31)
    _check_rne(np.concatenate([words, near]).view(np.float32))


def test_f16_widening_every_pattern():
    bits = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    got, want = F.f16_to_f32(bits), F.f16_bits_to_f32(bits)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))
    assert np.array_equal(F.f16_rne(got[~nan]), bits[~nan])  # round trip


def _inputs(world, n, seed, mode):
    rng = np.random.default_rng(seed)
    xs = []
    for r in range(world):
        x = (rng.standard_normal(n) * (1.0 if r % 2 else 300.0)).astype(np.float32)
        idx = rng.integers(0, n, size=n // 10)
        x[idx] = np.concatenate([TARGETED * 2, TARGETED])[rng.integers(0, 2 * TARGETED.size, size=idx.size)]
        xs.append(F.f32_to_f16_bits(x) if mode == F.B2O_F16 else x)
    return xs


@pytest.mark.parametrize("mode", [F.B2O_F32_WIRE_F16, F.B2O_F16])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_oracle_matches_numpy_twin(mode, world):
    for scale in (1.0 / world, 1.0, 1.0 / 3.0):
        xs = _inputs(world, 20_011, world * 10 + mode, mode)
        F.assert_f16_bits_equal(F.allreduce(mode, xs, scale), F.allreduce_numpy(mode, xs, scale), f"mode={mode} W={world} scale={scale}")


@pytest.mark.parametrize("mode", [F.B2O_F32_WIRE_F16, F.B2O_F16])
def test_oracle_matches_torch_restatement_at_w2(mode):
    """At W = 2 one fp32 add and one rounding to fp16 is the correctly rounded fp16 add: the reference's op sequence
    (cast, div_, fp16 SUM) gives the same bits as the oracle's fp32 accumulation."""
    xs = _inputs(2, 50_021, 3, mode)
    ts = [torch.from_numpy(x.view(np.int16)).view(torch.float16) if mode == F.B2O_F16 else torch.from_numpy(x) for x in xs]
    hook = "fp16_none" if mode == F.B2O_F16 else "fp16_compress"
    got = F.torch_hook_restatement(ts, hook)
    got = got.view(torch.int16).numpy().view(np.uint16) if mode == F.B2O_F16 else got.numpy()
    F.assert_f16_bits_equal(got, F.allreduce(mode, xs, 0.5), hook)


def test_oracle_matches_reference_ddp_w2_bit_exact():
    d = np.load(os.path.join(GOLDEN, "ddp_fp16_w2.npz"))
    want = F.allreduce(F.B2O_F32_WIRE_F16, list(d["local_f32"]), 0.5)
    want16 = F.allreduce(F.B2O_F16, list(d["local_f16"]), 0.5)
    for r in range(2):
        F.assert_f16_bits_equal(d["ddp_fp16_compress"][r], want, f"fp16_compress_hook, rank {r}")
        F.assert_f16_bits_equal(d["ddp_f16_none"][r], want16, f".half() model without a hook, rank {r}")


def test_oracle_within_w_minus_1_roundings_of_reference_ddp_w4():
    """At W = 4 gloo's own summation order and fp16 partial sums differ from the rank-order fp32 accumulation: within
    (W - 1) fp16 roundings, relative to the largest value of the bucket (partial sums can be larger than the result)."""
    W = 4
    d = np.load(os.path.join(GOLDEN, "ddp_fp16_w4.npz"))
    for key_in, key_out, mode in (("local_f32", "ddp_fp16_compress", F.B2O_F32_WIRE_F16), ("local_f16", "ddp_f16_none", F.B2O_F16)):
        want = F.allreduce(mode, list(d[key_in]), 1.0 / W)
        wf = (F.f16_bits_to_f32(want) if mode == F.B2O_F16 else want).astype(np.float64)
        for r in range(W):
            g = d[key_out][r]
            gf = (F.f16_bits_to_f32(g) if mode == F.B2O_F16 else g).astype(np.float64)
            rel = np.max(np.abs(gf - wf)) / np.max(np.abs(wf))
            assert 0 < rel < (W - 1) * 2.0 ** -11, (key_out, r, rel)  # > 0: the fixture really is a different order
        assert np.array_equal(d[key_out][0], d[key_out][W - 1])  # every rank holds the same bits


def test_header_constants_match_binding_and_oracle():
    with open(os.path.join(ROOT, "include", "b200ddp.h")) as f:
        src = f.read()

    def define(name):
        m = re.search(rf"#define\s+{name}\s+\(?(-?\d+)\)?", src)
        assert m, name
        return int(m.group(1))

    assert define("B2_F32_WIRE_F16") == N.B2_F32_WIRE_F16 == F.B2O_F32_WIRE_F16 == 3
    assert define("B2_F16") == N.B2_F16 == F.B2O_F16 == 4
    assert define("B2_ABI_VERSION") == N.B2_ABI_VERSION == N.lib().b2_version() == 3


@pytest.fixture
def _no_env_overrides(monkeypatch):
    for k in ("B2_ONESHOT_MAX_BYTES", "B2_PIPE_MIN_BYTES", "B2_NVLS_MIN_BYTES", "B2_NVLS_MIN_WORLD", "B2_LL_MIN_BYTES", "B2_LL_MAX_BYTES"):
        monkeypatch.delenv(k, raising=False)


@pytest.mark.usefixtures("_no_env_overrides")
def test_auto_policy_of_fp16_modes_is_the_bf16_wire_table():
    """AUTO is keyed on wire bytes: an fp16 wire takes exactly the bf16 wire's choices (NVLS at W = 8 from 64 MiB of wire
    data included), for the same number of 16-bit wire elements."""
    L = N.lib()
    sizes = [1, 4096, 100_003] + [int(m * MIB / 2) for m in (0.5, 1.0, 1.01, 4.0, 7.82, 8.0, 15.9, 16.0, 32.0, 63.9, 64.0, 512.0)]
    for world in range(1, 9):
        for mc in (0, 1):
            for n in sizes:
                want = L.b2_auto_algo(world, N.B2_F32_WIRE_BF16, n, mc)
                assert want >= 0
                assert L.b2_auto_algo(world, N.B2_F32_WIRE_F16, n, mc) == want, (world, mc, n)
                assert L.b2_auto_algo(world, N.B2_F16, n, mc) == want, (world, mc, n)
                assert L.b2_auto_algo(world, N.B2_BF16, n, mc) == want, (world, mc, n)
    n64 = 32 * MIB  # 16-bit wire elements in 64 MiB
    for mode in (N.B2_F32_WIRE_F16, N.B2_F16):
        assert L.b2_auto_algo(8, mode, n64, 1) == N.B2_ALGO_NVLS
        assert L.b2_auto_algo(8, mode, n64 - 8, 1) == N.B2_ALGO_TWOSHOT
        assert L.b2_auto_algo(8, mode, n64, 0) == N.B2_ALGO_TWOSHOT
        assert L.b2_auto_algo(4, mode, n64, 1) == N.B2_ALGO_TWOSHOT
    for bad in (5, 6, 7, -1):
        assert L.b2_auto_algo(2, bad, 100, 0) == N.B2_EINVAL


def test_mode_for_maps_dtype_and_wire():
    f32, f16, bf16 = torch.zeros(1), torch.zeros(1, dtype=torch.float16), torch.zeros(1, dtype=torch.bfloat16)
    assert mode_for(f32, "f16") == N.B2_F32_WIRE_F16
    assert mode_for(f32, "bf16") == N.B2_F32_WIRE_BF16 and mode_for(f32, "f32") == N.B2_F32
    for wire in ("f16", "bf16", "f32"):  # a 16-bit bucket is its own wire format
        assert mode_for(f16, wire) == N.B2_F16
        assert mode_for(bf16, wire) == N.B2_BF16
    with pytest.raises(ValueError):
        mode_for(f32, "f8")
    with pytest.raises(TypeError):
        mode_for(torch.zeros(1, dtype=torch.float64), "f16")


def test_fp16_hook_is_exported():
    import torchx_b200.ddp as ddp

    assert callable(ddp.b200_fp16_compress_hook)
