"""b2_reduce_scatter_step and ZeroRedundancyOptimizer(overlap_with_ddp=True) on the GPU, all ranks sharing one device.

Kernel: the fused step against torch._fused_sgd_ / _fused_adam_ / _fused_adamw_ on the oracle's block of the reduced
gradients (which reduce_scatter_gather_ into a shard must equal too), same slices, same hyper-parameters, parameters and
state bit for bit, the pad untouched.
Mini-DDP: overlap mode against the unsharded mini-DDP with the same optimizer class and fused=True, bit for bit after
every step and in the consolidated state; no_sync, checkpoints, the copy-in fallback and the run-time errors."""
import numpy as np
import pytest
import torch

from tests.test_zero_gpu import (WIRE, _assert_same, _assert_state_equal, _consolidate, _ddps, _input, _oracle, _params, _phase,
                                 _pieces, _warm, _world)
from torchx_b200.ddp import _native as N
from torchx_b200.ddp import zero as Z

pytestmark = pytest.mark.gpu

KINDS = {"sgd": N.B2_OPT_SGD, "adam": N.B2_OPT_ADAM, "adamw": N.B2_OPT_ADAMW}
# two groups of hyper-parameters per kind, with the options the fused kernels take
HYPER = {
    "sgd": [dict(lr=0.05, momentum=0.9, dampening=0.1, weight_decay=0.01, nesterov=False, maximize=False),
            dict(lr=0.02, momentum=0.8, dampening=0.0, weight_decay=0.0, nesterov=True, maximize=False)],
    "sgd0": [dict(lr=0.05, momentum=0.0, dampening=0.0, weight_decay=0.01, nesterov=False, maximize=False),
             dict(lr=0.02, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, maximize=True)],
    # maximize with momentum, with and without weight decay: checked on aligned parameters only (see below)
    "sgd_max": [dict(lr=0.05, momentum=0.9, dampening=0.0, weight_decay=0.0, nesterov=False, maximize=True),
                dict(lr=0.02, momentum=0.8, dampening=0.1, weight_decay=0.01, nesterov=True, maximize=True)],
    "adam": [dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, maximize=False),
             dict(lr=3e-3, beta1=0.8, beta2=0.99, eps=1e-6, weight_decay=0.0, maximize=True)],
}
HYPER["adamw"] = HYPER["adam"]
# torch's fused SGD contracts the momentum update of a maximized, undecayed gradient differently in its vectorised path
# (aligned tensors) and in its scalar path (the ragged slices here): SGD with maximize is checked on aligned parameters,
# in the mini-DDP tests below


def _table(kind, hyper, block, runs, param, s0, s1):
    t = N.B2Optim()
    t.kind, t.n_groups, t.n_runs = KINDS[kind.split("_")[0].rstrip("0")], len(hyper), len(runs)
    t.param, t.state0, t.state1 = param.data_ptr(), s0.data_ptr(), s1.data_ptr()
    for gi, h in enumerate(hyper):
        g = t.group[gi]
        for k, val in h.items():
            setattr(g, k, float(val) if not isinstance(val, bool) else int(val))
    for k, (lo, gi, st, *pos) in enumerate(runs):
        t.run_begin[k], t.run_group[k], t.run_step[k] = lo, gi, st
        if pos and pos[0] is not None:
            t.run_index[k], t.run_scalar[k] = pos[0]
    t.run_begin[len(runs)] = block
    return t


def _reference(kind, hyper, shard, P, M, V, runs, steps):
    """torch's fused optimizer over each run of this rank's block, one call per run (the kernels are elementwise)."""
    for (lo, hi, gi, i), step in zip(runs, steps):
        if gi == N.B2_OPT_NO_GROUP:
            continue
        h = hyper[gi]
        p, g, m, v = P[lo:hi], shard[lo:hi], M[lo:hi], V[lo:hi]
        if kind.startswith("sgd"):
            torch._fused_sgd_([p], [g], [m] if h["momentum"] else [], weight_decay=h["weight_decay"], momentum=h["momentum"],
                              lr=h["lr"], dampening=h["dampening"], nesterov=h["nesterov"], maximize=h["maximize"],
                              is_first_step=step == 0)
        else:
            fn = torch._fused_adam_ if kind == "adam" else torch._fused_adamw_
            st = torch.full((), float(step + 1), dtype=torch.float32, device="cuda")
            fn([p], [g], [m], [v], [], [st], lr=h["lr"], beta1=h["beta1"], beta2=h["beta2"], weight_decay=h["weight_decay"],
               eps=h["eps"], amsgrad=False, maximize=h["maximize"])


def _aligned_pieces(n, rng):
    """Parameter sizes of 16-element multiples (n is one): every run of every block is a 32-byte-aligned multiple of 8
    elements, so torch's fused kernels take their vectorised path on each slice."""
    sizes, left = [], n
    while left:
        k = int(min(left, 16 * rng.choice([1, 2, 5, 64, 700])))
        sizes.append(k)
        left -= k
    return sizes


def _check(W, mode, n, kind, seed, n_steps=3, stage_mb=8, adam_step0=0, aligned=False):
    w = _world(W, stage_mb)
    B = Z.padded_block(n, W)
    rng = np.random.default_rng(seed)
    sizes = _aligned_pieces(n, rng) if aligned else _pieces(n, rng, False)
    offsets = [sum(sizes[:i]) for i in range(len(sizes))]
    groups = [i % 2 for i in range(len(sizes))]  # neighbours in different groups, so groups meet inside vecs
    hyper = HYPER[kind]
    wire = WIRE[mode]
    tables, keep, xs = [], [], []
    for r in range(W):
        x = torch.randn(n, generator=torch.Generator().manual_seed(seed * 10 + r))
        xs.append(np.concatenate([x.numpy(), np.zeros(W * B - n, np.float32)]))
        x = x.cuda()
        segs = (N.B2Segment * (len(sizes) + 1))()
        for i, (o, k) in enumerate(zip(offsets, sizes)):
            off = 0 if aligned else i % 2
            t = torch.empty(k + off, device="cuda")[off:]  # every other gradient off a vec
            t.copy_(x[o:o + k])
            keep.append(t)
            segs[i].src, segs[i].begin, segs[i].end = t.data_ptr(), o, o + k
        nseg = len(sizes)
        if W * B > n:
            z = torch.zeros(W * B - n, device="cuda")
            keep.append(z)
            segs[nseg].src, segs[nseg].begin, segs[nseg].end = z.data_ptr(), n, W * B
            nseg += 1
        tables.append((segs, nseg))
    gen = torch.Generator().manual_seed(seed)
    P = [torch.randn(B, generator=gen).cuda() for _ in range(W)]
    M = [torch.randn(B, generator=gen).cuda() for _ in range(W)]
    V = [torch.rand(B, generator=gen).cuda() for _ in range(W)]
    ref = [(p.clone(), m.clone(), v.clone()) for p, m, v in zip(P, M, V)]
    runs = [Z.block_runs(offsets, sizes, groups, B, r) for r in range(W)]
    shards = [torch.empty(B, device="cuda") for _ in range(W)]
    # the reference steps the oracle's block, not the library's reduce-scatter: a reduction that both kernels got wrong
    # alike (a summation order, say) must not cancel out
    reduced = _oracle(mode, xs, 1.0 / W)
    blocks = [torch.from_numpy(reduced[r * B:(r + 1) * B].copy()).cuda() for r in range(W)]
    torch.cuda.synchronize()
    for step in range(adam_step0, adam_step0 + n_steps):
        counts = [[None if i is None else step for *_, i in rs] for rs in runs]
        # the reference steps each run as a tensor of its own: where an element sits in it, and whether the fused Adam
        # takes its scalar path there (a slice that is not 16-byte aligned or not a multiple of 4 elements)
        launch = [Z.launch_runs([(lo, gi, c, (0, lo % 4 != 0 or (hi - lo) % 4 != 0) if kind == "adam" else None)
                                 for (lo, hi, gi, _), c in zip(rs, cs)], kind.startswith("sgd"))
                  for rs, cs in zip(runs, counts)]
        opts = [_table(kind, hyper, B, launch[r], P[r], M[r], V[r]) for r in range(W)]
        w.run(lambda r, c, s: c.reduce_scatter_step_(B, tables[r][0], tables[r][1], opts[r], scale=1.0 / W, wire=wire, stream=s))
        w.run(lambda r, c, s: c.reduce_scatter_gather_(shards[r], tables[r][0], tables[r][1], scale=1.0 / W, wire=wire,
                                                       stream=s))
        for r in range(W):
            _reference(kind, hyper, blocks[r], *ref[r], runs[r], [step] * len(runs[r]))
        torch.cuda.synchronize()
        what = f"W={W} mode={mode} n={n} {kind} step {step}"
        for r in range(W):
            for name, got, want in zip("pmv", (P[r], M[r], V[r]), ref[r]):
                assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (
                    f"{what} rank {r} {name}: {(got != want).nonzero()[:8].flatten().tolist()}")
            assert torch.equal(shards[r].view(torch.int32), blocks[r].view(torch.int32)), f"{what} rank {r}: shard vs oracle"


@pytest.mark.parametrize("kind", ["sgd", "sgd0", "adam", "adamw"])
@pytest.mark.parametrize("mode", [0, 1, 3])
@pytest.mark.parametrize("W", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("n", [9, 4095, (1 << 17) + 3])
def test_step_matches_fused_optimizer(W, mode, n, kind):
    _check(W, mode, n, kind, seed=n % 89 + W)


@pytest.mark.parametrize("kind", ["sgd_max", "sgd", "adam", "adamw"])
@pytest.mark.parametrize("W", [1, 2, 4])
def test_step_matches_fused_optimizer_on_aligned_parameters(W, kind):
    # torch's fused SGD rounds the momentum update of a maximized, undecayed gradient differently in its vectorised path
    # (aligned tensors of 4-element multiples, what model parameters are) and its scalar path; ours is the vectorised one
    _check(W, 1, 16 * 3001, kind, seed=W + 40, aligned=True)


@pytest.mark.parametrize("W,mode,kind", [(2, 1, "adamw"), (2, 0, "sgd"), (4, 3, "adam")])
def test_block_larger_than_a_stage_region(W, mode, kind):
    n = 6_000_003  # stage_mb=8: several launches along the block axis
    assert Z.padded_block(n, W) * (4 if mode == 1 else 2) > (8 << 20) // (W + 1)
    _check(W, mode, n, kind, seed=3, n_steps=2)


def test_adam_bias_corrections_over_ten_thousand_steps():
    """powf of the library's CUDA against the fused Adam's, one run per step count: 128 counts per launch."""
    w = _world(1)
    n_runs, per = N.B2_OPT_MAX_RUNS, 8
    B = n_runs * per
    x = torch.randn(B, generator=torch.Generator().manual_seed(5)).cuda()
    segs = (N.B2Segment * 1)()
    segs[0].src, segs[0].begin, segs[0].end = x.data_ptr(), 0, B
    shard = torch.empty(B, device="cuda")
    w.run(lambda r, c, s: c.reduce_scatter_gather_(shard, segs, 1, scale=1.0, wire="f32", stream=s))
    for kind in ("adam", "adamw"):
        hyper = HYPER[kind]
        for first in range(1, 10_113, n_runs):
            P, M, V = torch.randn(B).cuda(), torch.randn(B).cuda(), torch.rand(B).cuda()
            want = [t.clone() for t in (P, M, V)]
            steps = list(range(first, first + n_runs))
            runs = [(k * per, k % 2, float(s), (0, False)) for k, s in enumerate(steps)]  # each run a tensor of 8
            opt = _table(kind, hyper, B, runs, P, M, V)
            w.run(lambda r, c, s: c.reduce_scatter_step_(B, segs, 1, opt, scale=1.0, wire="f32", stream=s))
            fn = torch._fused_adam_ if kind == "adam" else torch._fused_adamw_
            for gi in (0, 1):
                ks = [k for k in range(n_runs) if k % 2 == gi]
                sl = lambda t: [t[k * per:(k + 1) * per] for k in ks]  # noqa: E731
                h = hyper[gi]
                fn(sl(want[0]), sl(shard), sl(want[1]), sl(want[2]), [],
                   [torch.full((), float(steps[k]), device="cuda") for k in ks], lr=h["lr"], beta1=h["beta1"],
                   beta2=h["beta2"], weight_decay=h["weight_decay"], eps=h["eps"], amsgrad=False, maximize=h["maximize"])
            torch.cuda.synchronize()
            for got, ref in zip((P, M, V), want):
                assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), (kind, first)


# ---- the overlap mode of the mini-DDP -------------------------------------------------------------------------------
OPTS = {
    "sgd": (torch.optim.SGD, dict(lr=0.05, momentum=0.9, nesterov=True)),
    "sgd_maximize": (torch.optim.SGD, dict(lr=0.05, momentum=0.9, dampening=0.1, maximize=True)),
    "adam": (torch.optim.Adam, dict(lr=1e-3)),
    "adamw": (torch.optim.AdamW, dict(lr=1e-3)),
}


def _groups(ddp, cls=None):
    decay = [p for p in ddp.module.parameters() if p.dim() > 1]
    rest = [p for p in ddp.module.parameters() if p.dim() <= 1]
    first = {"params": decay, "weight_decay": 0.1}
    if cls is not torch.optim.SGD:
        first["eps"] = 1e-6
    return [first, {"params": rest, "weight_decay": 0.0, "lr": 2e-3}]


def _model(kind):
    from tests.test_zero_gpu import _conv, _mlp

    return _mlp if kind == "mlp" else _conv


def _run(W, opt, kind, steps=4, zero_copy=True, accumulate=False, checkpoint_at=None):
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    torch.backends.cudnn.deterministic = True
    cls, kw = OPTS[opt]
    ca, plain_ddps, sa = _ddps(W, _model(kind))
    cb, zero_ddps, sb = _ddps(W, _model(kind), zero_copy=zero_copy)
    try:
        plain = [cls(_groups(d, cls), fused=True, **kw) for d in plain_ddps]
        zero = [ZeroRedundancyOptimizer(d, cls, params=_groups(d, cls), overlap_with_ddp=True, fused=True, **kw) for d in zero_ddps]
        sched_p = [torch.optim.lr_scheduler.StepLR(o, step_size=2, gamma=0.5) for o in plain]
        sched_z = [torch.optim.lr_scheduler.StepLR(o, step_size=2, gamma=0.5) for o in zero]
        assert all(b.shard_grad is None for b in zero_ddps[0].buckets)  # no gradient shard in overlap mode

        def backward(r, step, ddp, o, s):
            with torch.cuda.stream(s):
                o.zero_grad()
                if accumulate:
                    with ddp.no_sync():
                        ddp(_input(kind, r, step + 50)).square().mean().backward()
                ddp(_input(kind, r, step)).square().mean().backward()

        def step_(o, sched, s):
            with torch.cuda.stream(s):
                o.step()
                sched.step()

        _warm(plain_ddps, sa, kind)
        _warm(zero_ddps, sb, kind)
        for step in range(steps):
            if step == checkpoint_at:  # consolidate; fresh models and overlap-mode optimizers load the checkpoint
                _consolidate(zero, 0, sb)
                sd = zero[0].state_dict()
                weights = [d.module.state_dict() for d in zero_ddps]
                cc, zero_ddps, sb = _ddps(W, _model(kind), zero_copy=zero_copy)
                cb += cc
                for d, wts in zip(zero_ddps, weights):
                    d.module.load_state_dict(wts)
                zero = [ZeroRedundancyOptimizer(d, cls, params=_groups(d, cls), overlap_with_ddp=True, fused=True, **kw)
                        for d in zero_ddps]
                for z in zero:
                    z.load_state_dict(sd)
                torch.cuda.synchronize()
                sched_z = [torch.optim.lr_scheduler.StepLR(o, step_size=2, gamma=0.5, last_epoch=step - 1) for o in zero]
                for o, p in zip(zero, plain):
                    for g, h in zip(o.param_groups, p.param_groups):
                        g["lr"] = h["lr"]
            _phase(W, lambda r: backward(r, step, plain_ddps[r], plain[r], sa[r]))
            _phase(W, lambda r: backward(r, step, zero_ddps[r], zero[r], sb[r]))
            _phase(W, lambda r: step_(plain[r], sched_p[r], sa[r]))
            _phase(W, lambda r: step_(zero[r], sched_z[r], sb[r]))
            for r in range(W):
                _assert_same(_params(zero_ddps[r]), _params(plain_ddps[r]), f"step {step} rank {r}")
        _consolidate(zero, 0, sb)
        _assert_state_equal(zero[0].state_dict(), plain[0].state_dict(), "consolidated state")
        return zero_ddps, zero, sb
    finally:
        for c in ca + cb:
            c.close()


@pytest.mark.parametrize("kind", ["mlp", "conv"])
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("W", [1, 2, 4])
def test_overlap_training_is_bit_equal_to_fused_unsharded(W, opt, kind):
    if W > 1:
        _run(1, opt, kind, steps=1)  # loads every compute kernel before the ranks wait on each other
    _run(W, opt, kind)


def test_overlap_no_sync_accumulation():
    _run(1, "adamw", "mlp", steps=1)
    _run(2, "adamw", "mlp", steps=3, accumulate=True)


def test_overlap_copy_in_fallback():
    _run(1, "sgd", "mlp", steps=1)
    _run(2, "sgd", "mlp", steps=3, zero_copy=False)
    _run(2, "adam", "conv", steps=3, zero_copy=False)


def test_overlap_checkpoint_round_trip():
    _run(1, "adamw", "mlp", steps=1)
    _run(2, "adamw", "mlp", steps=4, checkpoint_at=2)
    _run(2, "sgd", "mlp", steps=4, checkpoint_at=2)


def test_overlap_run_time_errors():
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    comms, ddps, ss = _ddps(1, _model("mlp"))
    try:
        d, s = ddps[0], ss[0]
        z = ZeroRedundancyOptimizer(d, torch.optim.AdamW, overlap_with_ddp=True, lr=1e-3)
        with torch.cuda.stream(s):
            z.step()  # no synced backward yet: a no-op
            assert not z._stepped
            d(_input("mlp", 0, 0)).square().mean().backward()
            with pytest.raises(RuntimeError, match="clip_grad_norm_"):
                z.clip_grad_norm_(1.0)
            with pytest.raises(RuntimeError, match="second synced backward before step"):
                d(_input("mlp", 0, 1)).square().mean().backward()
            scaler = torch.amp.GradScaler("cuda")
            with pytest.raises(RuntimeError, match="GradScaler"):
                z.step(grad_scaler=scaler)
            z.step()
            d(_input("mlp", 0, 2)).square().mean().backward()  # after step() a synced backward is fine again
            z.step()
        torch.cuda.synchronize()
    finally:
        for c in comms:
            c.close()
