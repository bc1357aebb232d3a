"""The layout of the model that tests/test_zero_position_gpu.py trains under ZeroRedundancyOptimizer, without a GPU: it stays
inside the contract (every bucket offset a multiple of 4 elements, 16 bytes) and rank blocks split a parameter whose numel
is not a multiple of 4 at the positions where torch's fused Adam rounds differently from a tensor of its own (DESIGN.md
2.4).  Checked here from the planner alone, so the GPU comparison cannot quietly stop reaching those positions."""
import pytest
import torch
from torch import nn

from torchx_b200.ddp import _native as N
from torchx_b200.ddp.bucketing import MIB, plan_buckets
from torchx_b200.ddp.zero import block_runs, padded_block

ODD_BIG = 61 * 2155  # 131455 = 3 (mod 4): torch's fused kernels step it on their scalar path
# W -> the indices in that weight where a rank block begins, other than 0
ODD_BOUNDARIES = {1: [], 2: [65728], 3: [43824, 87648], 4: [32864, 65728, 98592]}


def _odd(seed, device="cuda"):
    torch.manual_seed(seed)
    m = nn.Sequential(nn.Linear(33, 64), nn.ReLU(), nn.Linear(64, 61, bias=False), nn.ReLU(),
                      nn.Linear(61, 2155, bias=False), nn.ReLU(), nn.Linear(2155, 16))
    return m.to(device)


def _plan():
    """The buckets the mini-DDP of the GPU tests builds (bucket_cap_mb=0.01, first_bucket_mb=0.004)."""
    numels = [p.numel() for p in _odd(0, "cpu").parameters()]
    return plan_buckets(numels, [4] * len(numels), ["torch.float32"] * len(numels), int(0.004 * MIB), int(0.01 * MIB))


def test_odd_model_stays_inside_the_contract():
    specs = _plan()
    assert all(o % 4 == 0 for s in specs for o in s.offsets)
    big = [s for s in specs if ODD_BIG in s.numels]
    assert len(big) == 1 and big[0].numels == [ODD_BIG] and big[0].offsets == [0]  # alone, so nothing follows it off a vec
    assert [n % 4 for s in specs for n in s.numels].count(0) < len([n for s in specs for n in s.numels])


@pytest.mark.parametrize("W", [2, 3, 4])
def test_odd_model_block_boundaries_reach_the_scalar_path_slots(W):
    """Where each rank's run of the big weight begins in it: the positions the fused step must take into account, and the
    scalar-path slot (j % 2048) // 512 each one lands in (a tensor of its own would start in slot 0)."""
    (spec,) = [s for s in _plan() if ODD_BIG in s.numels]
    B = padded_block(spec.numel, W)
    starts = []
    for r in range(W):
        runs = [(lo, hi) for lo, hi, g, i in block_runs(spec.offsets, spec.numels, [0], B, r) if g != N.B2_OPT_NO_GROUP]
        starts += [lo + r * B - spec.offsets[0] for lo, _ in runs]
    assert starts == [0] + ODD_BOUNDARIES[W]
    slots = [(j % 2048) // 512 for j in ODD_BOUNDARIES[W]]
    assert slots == {2: [0], 3: [1, 3], 4: [0, 0, 0]}[W]
    assert all(j % 2048 != 0 for j in ODD_BOUNDARIES[W])  # counted from 0, every later run rounds some element otherwise
    if W == 2:
        assert ODD_BOUNDARIES[W][0] > 65536  # past the first 65536-element chunk


def _fake_ddp(W):
    """A DistributedDataParallel that was never constructed, with the odd model's bucket layout: enough for the checks
    that run before sharding."""
    from types import SimpleNamespace

    from torchx_b200.ddp import DistributedDataParallel

    m = _odd(0, "cpu")
    ps = list(m.parameters())
    d = DistributedDataParallel.__new__(DistributedDataParallel)
    for k, v in dict(module=m, _params=ps, wire="bf16", sharded=False, _synced_backwards=0, world_size=W,
                     buckets=[SimpleNamespace(spec=s, params=[ps[i] for i in s.param_indices]) for s in _plan()]).items():
        object.__setattr__(d, k, v)
    return d


def _groups(d, wd):
    return [{"params": [p for p in d._params if p.dim() > 1], "weight_decay": wd},
            {"params": [p for p in d._params if p.dim() <= 1], "weight_decay": 0.0}]


@pytest.mark.parametrize("W", [2, 3, 4])
def test_sharded_mode_refuses_fused_steps_that_depend_on_the_split(W):
    """Without overlap, torch's fused Adam with coupled decay and fused SGD with maximize, momentum and no decay would step
    the pieces of the split 131455-element weight to other bits than the whole tensor: refused before sharding, naming it."""
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    for cls, kw, wd, fix in ((torch.optim.Adam, dict(lr=1e-3, fused=True), 0.1, "overlap_with_ddp=True"),
                             (torch.optim.SGD, dict(lr=0.1, momentum=0.9, maximize=True, fused=True), 0.0, "foreach=True")):
        d = _fake_ddp(W)
        with pytest.raises(ValueError, match=r"parameter '4\.weight' \(131455 elements.*" + fix):
            ZeroRedundancyOptimizer(d, cls, params=_groups(d, wd), **kw)
        assert not d.sharded


@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_sharded_mode_accepts_what_steps_pieces_exactly(W):
    from torchx_b200.ddp import zero as Z

    d = _fake_ddp(W)
    ok = [(torch.optim.Adam, dict(fused=True), 0.0), (torch.optim.Adam, dict(fused=True, maximize=True), 0.1),
          (torch.optim.Adam, dict(foreach=True), 0.1), (torch.optim.Adam, {}, 0.1), (torch.optim.AdamW, dict(fused=True), 0.1),
          (torch.optim.SGD, dict(fused=True, momentum=0.9), 0.1), (torch.optim.SGD, dict(fused=True, maximize=True), 0.0),
          (torch.optim.SGD, dict(fused=True, maximize=True, momentum=0.9), 0.1),
          (torch.optim.SGD, dict(foreach=True, maximize=True, momentum=0.9), 0.0)]
    for cls, kw, wd in ok:
        Z._check_split_params(cls, _groups(d, wd), dict(lr=1e-3, **kw), d)
    if W == 1:  # one block: nothing is split
        Z._check_split_params(torch.optim.Adam, _groups(d, 0.1), dict(lr=1e-3, fused=True), d)
