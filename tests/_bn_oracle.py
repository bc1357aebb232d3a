"""numpy restatement of SyncBatchNorm's statistics merge: ATen's batch_norm_reduce_statistics_kernel<float, float, int32_t>
(torch/include/ATen/native/cuda/Normalization.cuh:459-502) with the contractions its SASS shows (DESIGN.md 2.4), every
operation rounded to fp32 on its own.  numpy's fp32 add, multiply, divide and sqrt are correctly rounded; the fused
multiply-adds are `fma32`."""
from __future__ import annotations

import numpy as np

f32 = np.float32


def fma32(a, b, c) -> np.ndarray:
    """Correctly rounded fp32 a * b + c.  The product is exact in fp64; the fp64 sum is rounded to odd (its exact error from
    TwoSum decides the last bit), after which the rounding to fp32 is correct: 53 >= 24 + 2 bits."""
    a, b, c = (np.asarray(x, dtype=np.float64) for x in np.broadcast_arrays(a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    even = (s.view(np.uint64) & 1) == 0
    fix = (err != 0) & even & np.isfinite(s)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def gather_stats(means, invstds, counts, running_mean=None, running_var=None, momentum=0.1, eps=1e-5):
    """(mean, invstd, running_mean, running_var) of torch.batch_norm_gather_stats_with_counts on the rows of the ranks with
    count >= 1 (torch's mask), in rank order.  means / invstds: [W, C] fp32, counts: [W] fp32.  The running statistics are
    returned updated (copies), or None when not given."""
    means = np.asarray(means, dtype=np.float32)
    invstds = np.asarray(invstds, dtype=np.float32)
    counts = np.asarray(counts, dtype=np.float32)
    eps, mom = f32(eps), f32(momentum)
    C = means.shape[1]
    avg = np.zeros(C, np.float32)
    var_n = np.zeros(C, np.float32)
    n = 0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for j in range(means.shape[0]):
            cnt = counts[j]
            if not cnt >= 1:
                continue
            nf = f32(n)
            x = f32(cnt + nf)
            factor = f32(f32(1) / x)
            v = f32(1) / invstds[j]
            a = fma32(v, v, -eps)
            d = avg - means[j]
            t = ((d * d) * nf * cnt) * factor
            var_n = var_n + fma32(a, cnt, t)
            avg = fma32(nf * factor, avg, means[j] * (cnt * factor))
            n = int(np.trunc(x))
        nf = f32(n)
        invstd = f32(1) / np.sqrt((var_n / nf) + eps)
        om = f32(1) - mom
        rm = rv = None
        if running_mean is not None:
            rm = fma32(avg, mom, om * np.asarray(running_mean, np.float32))
        if running_var is not None:
            rv = fma32(var_n / f32(n - 1), mom, om * np.asarray(running_var, np.float32))
    return avg.astype(np.float32), invstd.astype(np.float32), rm, rv


def local_stats(x: np.ndarray, eps: float):
    """One rank's (mean, invstd, count) of an [N, C] batch, computed in fp64 and rounded once: the test's stand-in for
    torch.batch_norm_stats."""
    x = np.asarray(x, dtype=np.float64)
    m = x.mean(axis=0)
    var = x.var(axis=0)
    return m.astype(np.float32), (1.0 / np.sqrt(var + eps)).astype(np.float32), np.float32(x.shape[0])
