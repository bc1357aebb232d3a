"""ZeroRedundancyOptimizer(overlap_with_ddp=True) without a GPU: the construction checks, the host tables of the fused
step (block runs, groups, step counts, the pad) and the argument checks of b2_reduce_scatter_step."""
import ctypes

import pytest
import torch

from torchx_b200.ddp import DistributedDataParallel
from torchx_b200.ddp import _native as N
from torchx_b200.ddp import zero as Z


def _fake_ddp(params, wire="bf16"):
    """A DistributedDataParallel that was never constructed: enough for the checks that run before sharding."""
    d = DistributedDataParallel.__new__(DistributedDataParallel)
    object.__setattr__(d, "_params", list(params))
    object.__setattr__(d, "wire", wire)
    object.__setattr__(d, "sharded", False)
    object.__setattr__(d, "_synced_backwards", 0)
    return d


def _refuses(exc, match, cls=torch.optim.AdamW, params=None, wire="bf16", **kw):
    ps = [torch.nn.Parameter(torch.zeros(4))] if params is None else params
    d = _fake_ddp(ps, wire)
    with pytest.raises(exc, match=match):
        Z.ZeroRedundancyOptimizer(d, cls, overlap_with_ddp=True, **kw)
    assert not d.sharded


def test_construction_errors_before_sharding():
    _refuses(ValueError, "amsgrad", lr=1e-3, amsgrad=True)
    _refuses(ValueError, "amsgrad", cls=torch.optim.Adam, lr=1e-3, amsgrad=True)
    _refuses(TypeError, "float lr", lr=torch.tensor(1e-3))
    _refuses(ValueError, "foreach", lr=1e-3, foreach=True)
    _refuses(ValueError, "capturable", lr=1e-3, capturable=True)
    _refuses(ValueError, "differentiable", lr=1e-3, differentiable=True)
    _refuses(ValueError, "foreach", cls=torch.optim.SGD, lr=0.1, foreach=True)
    _refuses(TypeError, "fp32 parameters", params=[torch.nn.Parameter(torch.zeros(4, dtype=torch.bfloat16))], lr=1e-3)
    _refuses(TypeError, "fp32 parameters", params=[torch.nn.Parameter(torch.zeros(4, dtype=torch.float16))], lr=1e-3)


def test_group_level_options_are_checked_too():
    a, b = torch.nn.Parameter(torch.zeros(4)), torch.nn.Parameter(torch.zeros(4))
    d = _fake_ddp([a, b])
    with pytest.raises(ValueError, match="amsgrad"):
        Z.ZeroRedundancyOptimizer(d, torch.optim.Adam, params=[{"params": [a]}, {"params": [b], "amsgrad": True}],
                                  overlap_with_ddp=True, lr=1e-3)
    ps = [torch.nn.Parameter(torch.zeros(2)) for _ in range(N.B2_OPT_MAX_GROUPS + 1)]
    with pytest.raises(ValueError, match="at most 8 parameter groups"):
        Z.ZeroRedundancyOptimizer(_fake_ddp(ps), torch.optim.SGD, params=[{"params": [p]} for p in ps],
                                  overlap_with_ddp=True, lr=0.1)


def test_constructed_after_a_backward_refuses():
    d = _fake_ddp([torch.nn.Parameter(torch.zeros(4))])
    object.__setattr__(d, "_synced_backwards", 1)
    with pytest.raises(RuntimeError, match="before the model's first backward"):
        Z.ZeroRedundancyOptimizer(d, torch.optim.SGD, overlap_with_ddp=True, lr=0.1)


def _runs_by_element(offsets, numels, groups, block, rank):
    """Restatement: the (group, parameter) of every element of rank's block, None past the bucket."""
    owner = {}
    for i, (o, n) in enumerate(zip(offsets, numels)):
        for e in range(o, o + n):
            owner[e] = (groups[i], i)
    return [owner.get(rank * block + e, (N.B2_OPT_NO_GROUP, None)) for e in range(block)]


@pytest.mark.parametrize("numels,groups", [
    ([1], [0]),
    ([7, 9], [0, 1]),
    ([3, 1, 100, 8, 8, 17], [0, 1, 1, 0, 2, 2]),  # groups alternate inside one vec
    ([64] * 9, [0, 1] * 4 + [0]),
    ([1000, 1, 1, 1, 333], [1, 0, 1, 0, 1]),
])
@pytest.mark.parametrize("W", [1, 2, 3, 4, 8])
def test_block_runs_tile_the_block(numels, groups, W):
    offsets = [sum(numels[:i]) for i in range(len(numels))]
    n_el = sum(numels)
    B = Z.padded_block(n_el, W)
    stepped = 0
    for r in range(W):
        runs = Z.block_runs(offsets, numels, groups, B, r)
        assert runs[0][0] == 0 and runs[-1][1] == B
        assert all(a[1] == b[0] for a, b in zip(runs, runs[1:]))  # contiguous, in order
        got = [(gi, i) for lo, hi, gi, i in runs for _ in range(lo, hi)]
        assert got == _runs_by_element(offsets, numels, groups, B, r)
        pad = [(lo, hi) for lo, hi, gi, i in runs if gi == N.B2_OPT_NO_GROUP]
        assert all(i is None for *_, i in runs if _[2] == N.B2_OPT_NO_GROUP)
        assert sum(hi - lo for lo, hi in pad) == max(0, min(B, (r + 1) * B - n_el))  # exactly the pad is excluded
        stepped += B - sum(hi - lo for lo, hi in pad)
    assert stepped == n_el


def test_launch_runs_steps_and_coalescing():
    # Adam: the update of a parameter that has taken n steps uses step n + 1; equal neighbours merge; the pad is 0
    runs = [(0, 0, 0), (5, 0, 0), (9, 1, 0), (12, 1, 3), (20, 0, 3), (30, Z.N.B2_OPT_NO_GROUP, None)]
    assert Z.launch_runs(runs, sgd=False) == [(0, 0, 1.0, None), (9, 1, 1.0, None), (12, 1, 4.0, None), (20, 0, 4.0, None),
                                              (30, 255, 0.0, None)]
    # SGD: 1.0 marks the first step (the momentum buffer starts as the gradient), 0.0 every later one
    assert Z.launch_runs(runs, sgd=True) == [(0, 0, 1.0, None), (9, 1, 1.0, None), (12, 1, 0.0, None), (20, 0, 0.0, None),
                                             (30, 255, 0.0, None)]
    # a run whose rounding depends on its place in its parameter (Adam's coupled weight decay) keeps its own entry
    assert Z.launch_runs([(0, 0, 0, (5, False)), (5, 0, 0, (0, True)), (9, 0, 0)], sgd=False) == [
        (0, 0, 1.0, (5, False)), (5, 0, 1.0, (0, True)), (9, 0, 1.0, None)]
    with pytest.raises(ValueError, match="alternates"):  # and counts on its own toward the table's bound
        Z._check_run_bound([[0] * 128], [[0] * 128], sgd=False, distinct=[[True] * 128])


def test_run_bound_is_checked_from_the_bucket_layout():
    # 127 runs of alternating groups and the pad fill the table; one more alternation does not fit, at any W
    Z._check_run_bound([[i % 2 for i in range(127)]], [[0] * 127], sgd=False)
    with pytest.raises(ValueError, match="alternates between parameter groups"):
        Z._check_run_bound([[i % 2 for i in range(128)]], [[0] * 128], sgd=False)
    Z._check_run_bound([[0] * 1000], [[0] * 1000], sgd=False)  # one group: one run, however many parameters
    with pytest.raises(ValueError, match="bucket 1"):  # step counts that differ split runs too
        Z._check_run_bound([[0], [0] * 200], [[0], list(range(200))], sgd=False)
    Z._check_run_bound([[0] * 200], [list(range(1, 201))], sgd=True)  # SGD only tells the first step from the others
    for W in (1, 2, 3, 8):  # a block never holds more runs than its bucket plus the pad
        numels = [3, 1, 100, 8, 8, 17, 5, 40]
        gs = [0, 1, 1, 0, 2, 2, 0, 1]
        offsets = [sum(numels[:i]) for i in range(len(numels))]
        B = Z.padded_block(sum(numels), W)
        bound = len(Z.launch_runs([(0, g, 0) for g in gs], False)) + 1
        for r in range(W):
            runs = Z.block_runs(offsets, numels, gs, B, r)
            assert len(Z.launch_runs([(lo, g, None if i is None else 0) for lo, _, g, i in runs], False)) <= bound


def test_kernel_bandwidth_counts_the_fused_pass_bytes():
    import importlib.util
    import os

    spec = importlib.util.spec_from_file_location(
        "zero_overlap_bench", os.path.join(os.path.dirname(N.INCLUDE_DIR), "tools", "zero_overlap_bench.py"))
    zb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(zb)
    assert zb.alg_bytes_per_element("adamw") == 4 + 12 + 12  # gradient read; parameter, exp_avg, exp_avg_sq read and written
    assert zb.alg_bytes_per_element("sgd") == 4 + 8 + 8


def _table(block=16, kind=N.B2_OPT_ADAMW, runs=((0, 0, 1.0),), groups=1):
    t = N.B2Optim()
    t.kind, t.n_groups, t.n_runs = kind, groups, len(runs)
    t.param, t.state0, t.state1 = 4096, 8192, 12288
    for k, (lo, gi, st) in enumerate(runs):
        t.run_begin[k], t.run_group[k], t.run_step[k] = lo, gi, st
    t.run_begin[len(runs)] = block
    for g in range(min(groups, N.B2_OPT_MAX_GROUPS)):
        t.group[g].lr, t.group[g].beta1, t.group[g].beta2, t.group[g].eps = 1e-3, 0.9, 0.999, 1e-8
    return t


def test_declared_and_bound():
    src = open(N.INCLUDE_DIR + "/b200ddp.h").read()
    assert "int b2_reduce_scatter_step(b2_comm_t* comm, size_t block, const b2_segment_t* segments" in src
    assert "b2_reduce_scatter_step" in N.SYMBOLS
    L = N.lib()
    assert L.b2_reduce_scatter_step.argtypes[6] is ctypes.POINTER(N.B2Optim)
    assert N.B2_ABI_VERSION == 3 == L.b2_version()


def test_einval_paths():
    L = N.lib()
    segs = (N.B2Segment * 1)()
    segs[0].src, segs[0].begin, segs[0].end = 4096, 0, 16

    def rc_of(t, mode=0, block=16):
        rc = L.b2_reduce_scatter_step(None, block, segs, 1, mode, 1.0, ctypes.byref(t) if t is not None else None, None)
        return rc, L.b2_last_error().decode()

    # the mode first, then block == 0 (a no-op), then the optimizer table, then the communicator
    for mode in (2, 4, 5, -1):
        assert rc_of(_table(), mode=mode) == (N.B2_EINVAL, f"b2_reduce_scatter_step: mode {mode} (fp32 buckets only: modes 0, 1, 3)")
    assert rc_of(None, block=0)[0] == N.B2_OK
    for mode in (0, 1, 3):
        assert rc_of(_table(), mode=mode) == (N.B2_EINVAL, "null communicator")
    assert rc_of(None) == (N.B2_EINVAL, "b2_reduce_scatter_step: null optimizer")
    assert rc_of(_table(kind=7)) == (N.B2_EINVAL, "b2_reduce_scatter_step: unknown optimizer kind 7")
    assert rc_of(_table(groups=9)) == (N.B2_EINVAL, "b2_reduce_scatter_step: need 1..8 parameter groups (got 9)")
    assert rc_of(_table(groups=0)) == (N.B2_EINVAL, "b2_reduce_scatter_step: need 1..8 parameter groups (got 0)")
    t = _table()
    t.n_runs = 0
    assert rc_of(t) == (N.B2_EINVAL, "b2_reduce_scatter_step: need 1..128 runs (got 0)")
    t = _table()
    t.state1 = None
    assert rc_of(t) == (N.B2_EINVAL, "b2_reduce_scatter_step: null parameter or state pointer")
    t = _table(kind=N.B2_OPT_SGD)
    t.state0 = t.state1 = None  # no group has momentum: no state is read
    assert rc_of(t) == (N.B2_EINVAL, "null communicator")
    t.group[0].momentum = 0.9
    assert rc_of(t) == (N.B2_EINVAL, "b2_reduce_scatter_step: null parameter or state pointer")
    t = _table()
    t.param = None
    assert rc_of(t) == (N.B2_EINVAL, "b2_reduce_scatter_step: null parameter or state pointer")
    t = _table(runs=((0, 0, 1.0), (8, 0, 1.0)))
    t.run_begin[2] = 15
    assert rc_of(t) == (N.B2_EINVAL, "b2_reduce_scatter_step: runs cover [0, 15), the block is [0, 16)")
    t = _table(runs=((0, 0, 1.0), (0, 0, 1.0)))
    assert rc_of(t) == (N.B2_EINVAL, "b2_reduce_scatter_step: run 0 is empty or out of order")
    assert rc_of(_table(runs=((0, 3, 1.0),))) == (N.B2_EINVAL, "b2_reduce_scatter_step: run 0 names group 3 of 1")
    assert rc_of(_table(runs=((0, N.B2_OPT_NO_GROUP, 0.0),)))[1] == "null communicator"  # an all-pad block is fine
    assert rc_of(_table(block=1 << 32), block=1 << 32)[1] == "b2_reduce_scatter_step: block of 4294967296 elements (the runs are 32-bit)"
