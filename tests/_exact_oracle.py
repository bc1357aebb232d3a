"""numpy oracle of the exact collectives (include/b200ddp.h: b2_allreduce_op MIN / MAX and integer SUM, b2_allgather).

Host forms: int32 / int64 arrays for the integer dtypes; raw bit patterns (uint32 for float32, uint16 for bfloat16 and
float16) for the float dtypes, so that every NaN payload and both zeros reach the kernels as they are."""
from __future__ import annotations

import functools
from typing import Sequence

import numpy as np

# dtype name -> (host dtype, bits, +inf bit pattern)
DTYPES = {
    "int32": (np.int32, 32, None),
    "int64": (np.int64, 64, None),
    "float32": (np.uint32, 32, 0x7F800000),
    "bfloat16": (np.uint16, 16, 0x7F80),
    "float16": (np.uint16, 16, 0x7C00),
}
CANONICAL_NAN = {"float32": 0x7FFFFFFF, "bfloat16": 0x7FFF, "float16": 0x7FFF}


def is_float(dtype: str) -> bool:
    return DTYPES[dtype][2] is not None


def isnan_bits(dtype: str, bits: np.ndarray) -> np.ndarray:
    _, nb, inf = DTYPES[dtype]
    u = bits.astype(np.uint64)
    return (u & ((1 << (nb - 1)) - 1)) > inf


def order_key(dtype: str, bits: np.ndarray) -> np.ndarray:
    """An unsigned key whose order is the IEEE total order on non-NaN values: -inf < ... < -0.0 < +0.0 < ... < +inf."""
    nb = DTYPES[dtype][1]
    u = bits.astype(np.uint64)
    sign = np.uint64(1 << (nb - 1))
    mask = np.uint64((1 << nb) - 1)
    return np.where(u & sign, ~u & mask, u | sign)


def reduce(dtype: str, op: str, inputs: Sequence[np.ndarray]) -> np.ndarray:
    """What every rank holds after b2_allreduce_op(dtype, op) of `inputs` (rank r's buffer = inputs[r]).  op is "sum"
    (integer dtypes only), "min" or "max".  A float result that is NaN comes back as the canonical NaN: the contract
    leaves the payload open (see assert_exact_equal)."""
    host, nb, _ = DTYPES[dtype]
    xs = [np.ascontiguousarray(x, dtype=host) for x in inputs]
    if not is_float(dtype):
        if op == "sum":  # two's complement: add as unsigned, wrap modulo 2^bits
            unsigned = np.uint32 if nb == 32 else np.uint64
            return functools.reduce(np.add, [x.view(unsigned) for x in xs]).view(host)
        if op in ("min", "max"):
            return (np.minimum if op == "min" else np.maximum).reduce(np.stack(xs), axis=0)
        raise ValueError(op)
    if op not in ("min", "max"):
        raise ValueError(f"{op} on {dtype} is not an exact op")
    stack = np.stack(xs)
    keys = order_key(dtype, stack)
    pick = np.argmin(keys, axis=0) if op == "min" else np.argmax(keys, axis=0)
    out = np.take_along_axis(stack, pick[None, :], axis=0)[0].copy()
    out[isnan_bits(dtype, stack).any(axis=0)] = CANONICAL_NAN[dtype]
    return out


def allgather(inputs: Sequence[np.ndarray]) -> np.ndarray:
    """Rank r's bytes at block r of the output."""
    return np.concatenate([np.ascontiguousarray(x).view(np.uint8).ravel() for x in inputs])


def assert_exact_equal(dtype: str, got: np.ndarray, want: np.ndarray, what: str = "") -> None:
    """Bit for bit, except that a NaN may carry any payload (the contract only promises that it is the same on every rank,
    which the callers check by comparing ranks with each other bit for bit)."""
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    if is_float(dtype):
        gn, wn = isnan_bits(dtype, got), isnan_bits(dtype, want)
        assert np.array_equal(gn, wn), f"{what}: NaN positions differ at {np.flatnonzero(gn != wn)[:8]}"
        bad = np.flatnonzero((got != want) & ~gn)
    else:
        bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: {bad.size} of {got.size} elements differ; first at {bad[:8]}: got {got[bad[:8]]} want {want[bad[:8]]}"
