"""ctypes front end of tests/oracle_f16.c (the CPU restatement of the fp16 modes), a numpy twin that restates it with
``np.float16`` independently, and test helpers for fp16 buckets.

The shared object is compiled on first use into the temporary directory (it is test infrastructure: the tree stays
untouched), named after a hash of the source so that an edited source is never served by a stale build."""
from __future__ import annotations

import ctypes
import hashlib
import os
import subprocess
import tempfile
from typing import Sequence

import numpy as np

B2O_F32_WIRE_F16 = 3
B2O_F16 = 4

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle_f16.c")
# the flags of oracle/Makefile: the oracle's roundings are part of the contract, so no contraction and no fast math
_CFLAGS = ["-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-std=c11", "-shared"]
_lib = None


def build() -> str:
    with open(_SRC, "rb") as f:
        digest = hashlib.sha256(f.read() + " ".join(_CFLAGS).encode()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"b2_oracle_f16_{os.getuid()}_{digest}.so")
    if not os.path.exists(so):
        fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(so))
        os.close(fd)
        try:
            subprocess.run([os.environ.get("CC", "gcc"), *_CFLAGS, "-o", tmp, _SRC], check=True)
            os.replace(tmp, so)
        finally:
            if os.path.exists(tmp):
                os.unlink(tmp)
    return so


def _load():
    global _lib
    if _lib is None:
        lib = ctypes.CDLL(build())
        lib.b2o_f16_allreduce.restype = ctypes.c_int
        lib.b2o_f16_allreduce.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_size_t,
                                          ctypes.c_float, ctypes.c_void_p]
        lib.b2o_f16_compress.restype = ctypes.c_int
        lib.b2o_f16_compress.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_float, ctypes.c_void_p]
        lib.b2o_f16_rne.restype = ctypes.c_uint16
        lib.b2o_f16_rne.argtypes = [ctypes.c_float]
        lib.b2o_f16_to_f32.restype = ctypes.c_float
        lib.b2o_f16_to_f32.argtypes = [ctypes.c_uint16]
        _lib = lib
    return _lib


def _elem_dtype(mode: int):
    if mode == B2O_F16:
        return np.uint16
    if mode == B2O_F32_WIRE_F16:
        return np.float32
    raise ValueError(f"not an fp16 mode: {mode}")


def allreduce(mode: int, inputs: Sequence[np.ndarray], scale: float) -> np.ndarray:
    """inputs[r]: rank r's bucket (float32 for mode 3, uint16 fp16 bit patterns for mode 4).  Returns the value every
    rank holds afterwards, same dtype."""
    lib = _load()
    dt = _elem_dtype(mode)
    arrs = [np.ascontiguousarray(a, dtype=dt) for a in inputs]
    n = arrs[0].size
    assert all(a.size == n for a in arrs)
    out = np.empty(n, dtype=dt)
    ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    rc = lib.b2o_f16_allreduce(mode, len(arrs), ptrs, n, ctypes.c_float(scale), out.ctypes.data)
    if rc != 0:
        raise ValueError(f"b2o_f16_allreduce rc={rc}")
    return out


def compress(mode: int, x: np.ndarray, scale: float) -> np.ndarray:
    """One rank's contribution c_r as fp32 values (all fp16-representable)."""
    lib = _load()
    x = np.ascontiguousarray(x, dtype=_elem_dtype(mode))
    out = np.empty(x.size, dtype=np.float32)
    if lib.b2o_f16_compress(mode, x.ctypes.data, x.size, ctypes.c_float(scale), out.ctypes.data) != 0:
        raise ValueError(mode)
    return out


def f16_rne(x: np.ndarray) -> np.ndarray:
    """fp32 values -> fp16 bits through the C oracle's conversion."""
    lib = _load()
    return np.array([lib.b2o_f16_rne(float(v)) for v in np.asarray(x, np.float32).ravel()], dtype=np.uint16)


def f16_to_f32(bits: np.ndarray) -> np.ndarray:
    lib = _load()
    return np.array([lib.b2o_f16_to_f32(int(b)) for b in np.asarray(bits, np.uint16).ravel()], dtype=np.float32)


# ---- numpy twin: np.float16 (IEEE binary16, round-to-nearest-even) as an independent restatement ------------------------
def f32_to_f16_bits(x: np.ndarray) -> np.ndarray:
    with np.errstate(all="ignore"):
        return np.ascontiguousarray(x, dtype=np.float32).astype(np.float16).view(np.uint16)


def f16_bits_to_f32(b: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(b, dtype=np.uint16).view(np.float16).astype(np.float32)


def allreduce_numpy(mode: int, inputs: Sequence[np.ndarray], scale: float) -> np.ndarray:
    sc = np.float32(scale)
    acc = None
    with np.errstate(all="ignore"):
        for a in inputs:
            v = f16_bits_to_f32(a) if mode == B2O_F16 else f16_bits_to_f32(f32_to_f16_bits(a))
            c = f16_bits_to_f32(f32_to_f16_bits((v * sc).astype(np.float32)))
            acc = c if acc is None else (acc + c).astype(np.float32)
    bits = f32_to_f16_bits(acc)
    return bits if mode == B2O_F16 else f16_bits_to_f32(bits)


def torch_hook_restatement(inputs, hook: str):
    """The reference's own op sequence on CPU torch tensors, reduced in rank order with an fp16 rounding after every add
    (what a ring would do).  hook: "fp16_compress" (fp32 gradients, default_hooks.fp16_compress_hook) or "fp16_none"
    (fp16 gradients, no hook: pre-divide, SUM in fp16)."""
    import torch

    if hook not in ("fp16_compress", "fp16_none"):
        raise ValueError(hook)
    w = len(inputs)
    acc = None
    for g in inputs:
        c = g.to(torch.float16, copy=True).div_(w)  # copy: an fp16 `g` would otherwise be divided in place
        acc = c if acc is None else acc + c  # fp16 + fp16 -> rounds to fp16 each step
    return acc.float() if hook == "fp16_compress" else acc


# ---- test helpers -------------------------------------------------------------------------------------------------------
def assert_f16_bits_equal(got: np.ndarray, want: np.ndarray, what: str = "") -> None:
    """Bit-exact comparison of fp16 buckets (uint16 bits) or fp32 buckets holding fp16 values; NaNs must coincide but their
    payloads may differ."""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.dtype == np.uint16:
        gf, wf = f16_bits_to_f32(got), f16_bits_to_f32(want)
        gi, wi = got, want
    else:
        gf, wf = got.astype(np.float32, copy=False), want.astype(np.float32, copy=False)
        gi, wi = gf.view(np.uint32), wf.view(np.uint32)
    gn, wn = np.isnan(gf), np.isnan(wf)
    assert np.array_equal(gn, wn), f"{what}: NaN positions differ at {np.flatnonzero(gn != wn)[:8]}"
    bad = np.flatnonzero((gi != wi) & ~gn)
    assert bad.size == 0, (
        f"{what}: {bad.size} of {got.size} elements differ; first at {bad[:8]}: got {gf[bad[:8]]} want {wf[bad[:8]]}")


def f16_ulp(v: np.ndarray) -> np.ndarray:
    """One fp16 ulp at |v| (float64): 2^(e - 10) for normals, 2^-24 for subnormals."""
    a = np.abs(np.asarray(v, np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 10)


def assert_nvls_f16_result(got: np.ndarray, inputs: list, scale: float, mode: int, what: str = "") -> dict:
    """The NVSwitch adds the W fp16 contributions with fp32 accumulation and one rounding, in its own order.  Contract:
    equal to the rank-order oracle wherever that is order-independent, and everywhere within one fp16 ulp of the exact
    (float64) sum of the contributions."""
    want = allreduce(mode, inputs, scale)
    exact = np.sum([compress(mode, x, scale).astype(np.float64) for x in inputs], axis=0)
    gf = f16_bits_to_f32(got) if got.dtype == np.uint16 else got.astype(np.float32)
    wf = f16_bits_to_f32(want) if want.dtype == np.uint16 else want.astype(np.float32)
    gn, wn = np.isnan(gf), np.isnan(wf)
    assert np.array_equal(gn, wn), f"{what}: NaN positions differ at {np.flatnonzero(gn != wn)[:8]}"
    diff = np.flatnonzero((gf.view(np.uint32) != wf.view(np.uint32)) & ~gn)
    if diff.size:
        err = np.abs(gf[diff].astype(np.float64) - exact[diff])
        fin = np.isfinite(exact[diff]) & (np.abs(exact[diff]) < 65504.0)
        bad = diff[(err > f16_ulp(exact[diff])) & fin]
        assert bad.size == 0, (f"{what}: {bad.size} elements are more than one fp16 ulp from the exact sum; first at {bad[:8]}: "
                               f"got {gf[bad[:8]]} exact {exact[bad[:8]]} rank-order {wf[bad[:8]]}")
    return {"n": int(got.size), "differ_from_rank_order": int(diff.size)}
