"""ZeroRedundancyOptimizer(master_weights=True) without a GPU: the keyword, its refusals and their order, the fused step's
table over the masters of a bf16 bucket, the argument checks of b2_reduce_scatter_step_bf16 and the byte counts of
tools/zero_master_bench.py."""
import ctypes
import importlib.util
import inspect
import os
import types

import pytest
import torch

from torchx_b200.ddp import DistributedDataParallel
from torchx_b200.ddp import _native as N
from torchx_b200.ddp import zero as Z


def _fake_ddp(params, wire="bf16", find_unused=False):
    """A DistributedDataParallel that was never constructed: enough for the checks that run before sharding."""
    d = DistributedDataParallel.__new__(DistributedDataParallel)
    object.__setattr__(d, "_params", list(params))
    object.__setattr__(d, "wire", wire)
    object.__setattr__(d, "sharded", False)
    object.__setattr__(d, "_synced_backwards", 0)
    object.__setattr__(d, "find_unused_parameters", find_unused)
    return d


def _p(dtype, n=4):
    return torch.nn.Parameter(torch.zeros(n, dtype=dtype))


def test_keyword_defaults_to_off():
    sig = inspect.signature(Z.ZeroRedundancyOptimizer.__init__)
    assert sig.parameters["master_weights"].default is False
    # without the flag, bf16 parameters are refused by overlap mode as before, with the old text
    d = _fake_ddp([_p(torch.bfloat16)])
    with pytest.raises(TypeError, match=r"overlap_with_ddp=True steps fp32 parameters only \(modes B2_F32_WIRE_BF16"):
        Z.ZeroRedundancyOptimizer(d, torch.optim.AdamW, overlap_with_ddp=True, lr=1e-3)


@pytest.mark.parametrize("overlap", [False, True])
def test_refusals(overlap):
    d = _fake_ddp([_p(torch.bfloat16), _p(torch.float16)])
    with pytest.raises(TypeError, match="master_weights=True keeps fp32 masters for bf16 parameters only"):
        Z.ZeroRedundancyOptimizer(d, torch.optim.AdamW, overlap_with_ddp=overlap, master_weights=True, lr=1e-3)
    d = _fake_ddp([_p(torch.float32)])
    with pytest.raises(ValueError, match="master_weights=True needs bf16 parameters: the model has none"):
        Z.ZeroRedundancyOptimizer(d, torch.optim.AdamW, overlap_with_ddp=overlap, master_weights=True, lr=1e-3)
    assert not d.sharded


def test_existing_refusals_come_first():
    fp16 = [_p(torch.float16)]  # would be refused by master_weights
    with pytest.raises(TypeError, match="ZeroRedundancyOptimizer supports"):
        Z.ZeroRedundancyOptimizer(_fake_ddp(fp16), torch.optim.RMSprop, master_weights=True, lr=1e-3)
    with pytest.raises(TypeError, match="shards a torchx_b200.ddp.DistributedDataParallel"):
        Z.ZeroRedundancyOptimizer(torch.nn.Linear(2, 2), torch.optim.AdamW, master_weights=True, lr=1e-3)
    with pytest.raises(ValueError, match="cannot be combined with find_unused_parameters=True"):
        Z.ZeroRedundancyOptimizer(_fake_ddp(fp16, find_unused=True), torch.optim.AdamW, overlap_with_ddp=True,
                                  master_weights=True, lr=1e-3)
    with pytest.raises(ValueError, match="in no parameter group"):
        Z.ZeroRedundancyOptimizer(_fake_ddp(fp16 + [_p(torch.bfloat16)]), torch.optim.AdamW, params=fp16,
                                  master_weights=True, lr=1e-3)


def test_overlap_checks_still_apply_with_masters():
    ps = [_p(torch.bfloat16), _p(torch.float32)]
    for kw, exc, match in [(dict(amsgrad=True), ValueError, "amsgrad"), (dict(foreach=True), ValueError, "foreach"),
                           (dict(lr=torch.tensor(1e-3)), TypeError, "float lr")]:
        d = _fake_ddp(ps)
        with pytest.raises(exc, match=match):
            Z.ZeroRedundancyOptimizer(d, torch.optim.AdamW, overlap_with_ddp=True, master_weights=True,
                                      **{"lr": 1e-3, **kw})
        assert not d.sharded
    d = _fake_ddp(ps)
    object.__setattr__(d, "_synced_backwards", 1)
    with pytest.raises(RuntimeError, match="before the model's first backward"):
        Z.ZeroRedundancyOptimizer(d, torch.optim.AdamW, overlap_with_ddp=True, master_weights=True, lr=1e-3)


def _stand_in(numels, world, rank, overlap, dtype=torch.bfloat16):
    """A ZeroRedundancyOptimizer over a one-bucket stand-in model on the CPU, built without its constructor's sharding."""
    from torchx_b200.ddp.bucketing import MIB, plan_buckets

    params = [torch.nn.Parameter(torch.randn(n).to(dtype)) for n in numels]
    (spec,) = plan_buckets(numels, [params[0].element_size()] * len(numels), [str(dtype)] * len(numels), MIB, MIB)
    block = Z.padded_block(spec.numel, world)
    b = types.SimpleNamespace(spec=spec, params=[params[i] for i in spec.param_indices], dtype=dtype, block=block,
                              param_flat=torch.zeros(world * block, dtype=dtype),
                              shard_grad=None if overlap else torch.zeros(block, dtype=dtype))
    for p, o, n in zip(b.params, spec.offsets, spec.numels):
        b.param_flat[o:o + n] = p.data
        p.data = b.param_flat[o:o + n]
    model = types.SimpleNamespace(buckets=[b], device=torch.device("cpu"), world_size=world, _shard_grads=[],
                                  comm=types.SimpleNamespace(rank=rank), _params=params)
    model._enable_sharding = lambda zero: None
    model._check_shardable = lambda: None
    model.module = torch.nn.Module()
    model.wire = "bf16"
    model.find_unused_parameters = False
    orig = Z.DistributedDataParallel
    Z.DistributedDataParallel = types.SimpleNamespace  # the stand-in passes the isinstance check
    try:
        groups = [{"params": params[0::2]}, {"params": params[1::2], "lr": 2e-3}]
        z = Z.ZeroRedundancyOptimizer(model, torch.optim.AdamW, params=groups, overlap_with_ddp=overlap,
                                      master_weights=True, lr=1e-3)
    finally:
        Z.DistributedDataParallel = orig
    return z, b, model


@pytest.mark.parametrize("W,rank", [(1, 0), (2, 1), (3, 2)])
def test_masters_and_the_launch_table_of_a_bf16_bucket(W, rank):
    numels = [7, 9, 100, 3, 41]
    z, b, model = _stand_in(numels, W, rank, overlap=True)
    B = b.block
    m = z._master_flat[0]
    assert m.dtype == torch.float32 and m.numel() == B  # this rank's block only
    assert torch.equal(m, b.param_flat[rank * B:(rank + 1) * B].float())  # the exact widening
    # the inner optimizer steps 1-D fp32 views of the masters, one per (parameter, this rank's block)
    views = [v for g in z.param_groups for v in g["params"]]
    assert views and all(v.dtype == torch.float32 and v.dim() == 1 and v.untyped_storage().data_ptr() == m.data_ptr()
                         for v in views)
    t = z._launch_table(b)
    assert t.param == m.data_ptr()  # the masters, not the bf16 parameters
    assert t.state0 == z._flat_state[0]["exp_avg"].data_ptr() and t.state1 == z._flat_state[0]["exp_avg_sq"].data_ptr()
    assert all(s.dtype == torch.float32 and s.numel() == B for s in z._flat_state[0].values())
    runs = Z.block_runs(b.spec.offsets, b.spec.numels, [i % 2 for i in b.spec.param_indices], B, rank)
    want = Z.launch_runs([(lo, gi, None if i is None else 0) for lo, _, gi, i in runs], sgd=False)
    assert t.n_runs == len(want)
    assert [(t.run_begin[k], t.run_group[k], t.run_step[k]) for k in range(t.n_runs)] == [(lo, gi, st) for lo, gi, st, _ in want]
    assert t.run_begin[t.n_runs] == B


def test_without_overlap_the_inner_optimizer_reads_fp32_gradient_blocks():
    z, b, model = _stand_in([7, 9, 100], 2, 0, overlap=False)
    g = z._master_grad[0]
    assert g.dtype == torch.float32 and g.numel() == b.block
    assert model._shard_widen == [(b.shard_grad, g)]
    for v, grad, p in model._shard_grads:
        assert v.dtype == torch.float32 and grad.dtype == torch.float32 and grad.untyped_storage().data_ptr() == g.data_ptr()


def test_an_fp32_only_model_is_refused():
    with pytest.raises(ValueError, match="needs bf16 parameters"):
        _stand_in([7, 9], 1, 0, overlap=True, dtype=torch.float32)


def _table(block=16):
    t = N.B2Optim()
    t.kind, t.n_groups, t.n_runs = N.B2_OPT_ADAMW, 1, 1
    t.param, t.state0, t.state1 = 4096, 8192, 12288
    t.run_begin[0], t.run_group[0], t.run_step[0], t.run_begin[1] = 0, 0, 1.0, block
    t.group[0].lr, t.group[0].beta1, t.group[0].beta2, t.group[0].eps = 1e-3, 0.9, 0.999, 1e-8
    return t


def test_declared_and_bound():
    src = open(N.INCLUDE_DIR + "/b200ddp.h").read()
    assert ("int b2_reduce_scatter_step_bf16(b2_comm_t* comm, size_t block, const b2_segment_t* segments, int n_segments, "
            "float scale,") in src
    assert "b2_reduce_scatter_step_bf16" in N.SYMBOLS
    L = N.lib()
    assert L.b2_reduce_scatter_step_bf16.argtypes[5] is ctypes.POINTER(N.B2Optim)
    assert N.B2_ABI_VERSION == 3 == L.b2_version()


def test_einval_paths():
    L = N.lib()
    segs = (N.B2Segment * 1)()
    segs[0].src, segs[0].begin, segs[0].end = 4096, 0, 16
    fn = "b2_reduce_scatter_step_bf16"

    def rc_of(t, block=16, pbf=16384):
        rc = L.b2_reduce_scatter_step_bf16(None, block, segs, 1, 1.0, ctypes.byref(t) if t is not None else None, pbf, None)
        return rc, L.b2_last_error().decode()

    assert rc_of(None, block=0)[0] == N.B2_OK  # block == 0 is a no-op
    assert rc_of(_table()) == (N.B2_EINVAL, "null communicator")
    assert rc_of(None) == (N.B2_EINVAL, f"{fn}: null optimizer")
    t = _table()
    t.kind = 7
    assert rc_of(t) == (N.B2_EINVAL, f"{fn}: unknown optimizer kind 7")
    t = _table()
    t.n_groups = 9
    assert rc_of(t) == (N.B2_EINVAL, f"{fn}: need 1..8 parameter groups (got 9)")
    t = _table()
    t.n_runs = 0
    assert rc_of(t) == (N.B2_EINVAL, f"{fn}: need 1..128 runs (got 0)")
    t = _table()
    t.state1 = None
    assert rc_of(t) == (N.B2_EINVAL, f"{fn}: null parameter or state pointer")
    t = _table()
    t.param = None
    assert rc_of(t) == (N.B2_EINVAL, f"{fn}: null parameter or state pointer")
    t = _table()
    t.run_begin[1] = 15
    assert rc_of(t) == (N.B2_EINVAL, f"{fn}: runs cover [0, 15), the block is [0, 16)")
    t = _table()
    t.run_group[0] = 3
    assert rc_of(t) == (N.B2_EINVAL, f"{fn}: run 0 names group 3 of 1")
    assert rc_of(_table(), pbf=None) == (N.B2_EINVAL, f"{fn}: null bf16 parameter pointer")
    assert rc_of(_table(), pbf=16384 + 8) == (N.B2_EINVAL, f"{fn}: bf16 parameter pointer not 16-byte aligned")
    assert rc_of(_table(1 << 32), block=1 << 32)[1] == f"{fn}: block of 4294967296 elements (the runs are 32-bit)"


def _bench():
    spec = importlib.util.spec_from_file_location(
        "zero_master_bench", os.path.join(os.path.dirname(N.INCLUDE_DIR), "tools", "zero_master_bench.py"))
    zb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(zb)
    return zb


def test_bench_byte_counts():
    zb = _bench()
    assert zb.alg_bytes_per_element(master=False) == 4 + 12 + 12
    assert zb.alg_bytes_per_element(master=True) == 2 + 12 + 12 + 2
    numels = [1000, 3, 50_000, 7]
    for W in (1, 2, 4):
        fp32 = zb.bytes_per_rank(numels, 4, W, masters=False)
        bf16 = zb.bytes_per_rank(numels, 2, W, masters=True)
        B = Z.padded_block(sum(numels), W)  # one bucket either way at these sizes
        assert fp32["param_bytes"] == 4 * W * B and fp32["state_bytes"] == 8 * B and fp32["master_bytes"] == 0
        assert bf16["param_bytes"] == 2 * W * B and bf16["state_bytes"] == 8 * B and bf16["master_bytes"] == 4 * B
        assert bf16["total_bytes"] == 2 * W * B + 12 * B and fp32["total_bytes"] == 4 * W * B + 8 * B
