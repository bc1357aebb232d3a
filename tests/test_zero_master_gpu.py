"""ZeroRedundancyOptimizer(master_weights=True) and b2_reduce_scatter_step_bf16 on the GPU, all ranks sharing one device.

Kernel: the fused bf16 step against the oracle's bf16 reduce-scatter, widened, then torch's fused SGD / Adam / AdamW on
fp32 copies of the masters and state, then ``.to(torch.bfloat16)`` on the device (ATen's CUDA conversion, which the
training reference's ``param.copy_(master)`` makes): masters, state and bf16 parameters bit for bit, the pad untouched.
Mini-DDP: a bf16 model (one fp32 parameter left in it) against the unsharded mini-DDP over the same model with hand-held
fp32 masters, bit for bit in the bf16 parameters, the masters and the consolidated state."""
import numpy as np
import pytest
import torch
from torch import nn

from tests.test_zero_gpu import _assert_state_equal, _consolidate, _ddps, _host, _phase, _pieces, _world
from tests.test_zero_overlap_gpu import HYPER, _reference, _table
from torchx_b200.ddp import _native as N
from torchx_b200.ddp import zero as Z

pytestmark = pytest.mark.gpu


def _bits(t):
    t = t.detach().contiguous().cpu()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _assert_bits(got, want, what):
    g, w = _bits(got), _bits(want)
    assert g.shape == w.shape and torch.equal(g, w), f"{what}: {(g != w).nonzero()[:8].flatten().tolist()}"


# ---- the kernel -----------------------------------------------------------------------------------------------------
def _check(W, n, kind, seed, n_steps=3, stage_mb=8, specials=False):
    import oracle

    w = _world(W, stage_mb)
    B = Z.padded_block(n, W)
    rng = np.random.default_rng(seed)
    sizes = _pieces(n, rng, False)
    offsets = [sum(sizes[:i]) for i in range(len(sizes))]
    groups = [i % 2 for i in range(len(sizes))]
    hyper = HYPER[kind]
    runs = [Z.block_runs(offsets, sizes, groups, B, r) for r in range(W)]
    gen = torch.Generator().manual_seed(seed)
    masters = [torch.randn(B, generator=gen).cuda() for _ in range(W)]
    if specials:  # the conversion of NaN and +-inf masters
        for m in masters:
            m[1], m[2], m[3] = float("nan"), float("inf"), -float("inf")
            m[5] = -float("nan")
    M = [torch.randn(B, generator=gen).cuda() for _ in range(W)]
    V = [torch.rand(B, generator=gen).cuda() for _ in range(W)]
    pbf = [torch.full((W * B,), 7.0, dtype=torch.bfloat16, device="cuda") for _ in range(W)]  # the whole bucket
    ref = [(m.clone(), a.clone(), v.clone()) for m, a, v in zip(masters, M, V)]
    for step in range(n_steps):
        xs, tables, keep = [], [], []
        for r in range(W):
            x = torch.randn(n, generator=torch.Generator().manual_seed(seed * 100 + step * 10 + r)).bfloat16().cuda()
            xs.append(x)
            segs = (N.B2Segment * (len(sizes) + 2))()
            nseg = 0
            for i, (o, k) in enumerate(zip(offsets, sizes)):
                if i % 7 == 3:  # a zero segment (an unused parameter)
                    segs[nseg].src = N.B2_SEGMENT_ZEROS
                    x[o:o + k] = 0
                else:
                    t = torch.empty(k + i % 2, dtype=torch.bfloat16, device="cuda")[i % 2:]  # every other one off a vec
                    t.copy_(x[o:o + k])
                    keep.append(t)
                    segs[nseg].src = t.data_ptr()
                segs[nseg].begin, segs[nseg].end = o, o + k
                nseg += 1
            if W * B > n:
                z = torch.zeros(W * B - n, dtype=torch.bfloat16, device="cuda")
                keep.append(z)
                segs[nseg].src, segs[nseg].begin, segs[nseg].end = z.data_ptr(), n, W * B
                nseg += 1
            tables.append((segs, nseg))
        launch = [Z.launch_runs([(lo, gi, None if i is None else step,
                                  (0, lo % 4 != 0 or (hi - lo) % 4 != 0) if kind == "adam" else None)
                                 for lo, hi, gi, i in rs], kind.startswith("sgd")) for rs in runs]
        opts = [_table(kind, hyper, B, launch[r], masters[r], M[r], V[r]) for r in range(W)]
        torch.cuda.synchronize()
        w.run(lambda r, c, s: c.reduce_scatter_step_bf16_(B, tables[r][0], tables[r][1], opts[r], pbf[r][r * B:(r + 1) * B],
                                                          scale=1.0 / W, stream=s))
        # the reference: the oracle's bf16 reduce-scatter, widened, and torch's fused step on fp32 copies
        want = oracle.allreduce(N.B2_BF16, [_host(x) for x in xs], 1.0 / W)
        full = np.zeros(W * B, dtype=np.uint16)
        full[:n] = want
        for r in range(W):
            shard = torch.from_numpy(full[r * B:(r + 1) * B].astype(np.int16)).view(torch.bfloat16).float().cuda()
            _reference(kind, hyper, shard, *ref[r], runs[r], [step] * len(runs[r]))
        torch.cuda.synchronize()
        what = f"W={W} n={n} {kind} step {step}"
        for r in range(W):
            for name, got, exp in zip(("master", "state0", "state1"), (masters[r], M[r], V[r]), ref[r]):
                _assert_bits(got, exp, f"{what} rank {r} {name}")
            stepped = torch.zeros(B, dtype=torch.bool)
            for lo, hi, gi, _ in runs[r]:
                stepped[lo:hi] = gi != N.B2_OPT_NO_GROUP
            got = pbf[r][r * B:(r + 1) * B].cpu()
            conv = ref[r][0].to(torch.bfloat16).cpu()  # ATen's conversion on the device
            _assert_bits(got[stepped], conv[stepped], f"{what} rank {r} bf16 parameters")
            seven = torch.full((W * B,), 7.0, dtype=torch.bfloat16)
            _assert_bits(got[~stepped], seven[:B][~stepped], f"{what} rank {r}: the pad is not written")
            outside = torch.cat([pbf[r][:r * B], pbf[r][(r + 1) * B:]]).cpu()
            _assert_bits(outside, seven[:outside.numel()], f"{what} rank {r}: only this rank's block is written")
            if specials and r == 0:
                assert stepped[1] and stepped[5] and torch.isnan(got[[1, 5]]).all()


# SGD with maximize, momentum and no weight decay is left out: the per-run reference steps unaligned slices on the fused
# SGD's scalar path, which contracts its momentum update differently (DESIGN.md 2.4); the mini-DDP tests cover maximize
@pytest.mark.parametrize("kind", ["sgd", "sgd0", "adam", "adamw"])
@pytest.mark.parametrize("W", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("n", [9, 4095, 16 * 4096, (1 << 17) + 3])
def test_bf16_step_matches_oracle_and_fused_optimizer(W, n, kind):
    _check(W, n, kind, seed=n % 89 + W)


@pytest.mark.parametrize("W", [1, 2])
def test_bf16_step_converts_nan_and_inf_as_aten(W):
    _check(W, 4095, "sgd0", seed=17, n_steps=1, specials=True)


@pytest.mark.parametrize("W,kind", [(2, "adamw"), (4, "sgd")])
def test_bf16_step_block_larger_than_a_stage_region(W, kind):
    n = 6_000_003  # stage_mb=8: several launches along the block axis
    assert Z.padded_block(n, W) * 2 > (8 << 20) // (W + 1)
    _check(W, n, kind, seed=3, n_steps=2)


# ---- the mini-DDP ---------------------------------------------------------------------------------------------------
class _Mlp(nn.Module):
    def __init__(self, seed):
        super().__init__()
        torch.manual_seed(seed)
        self.body = nn.Sequential(nn.Linear(33, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 16))
        self.body.bfloat16()
        self.gain = nn.Parameter(torch.ones(16))  # left in fp32

    def forward(self, x):
        return self.body(x).float() * self.gain


class _Conv(nn.Module):
    def __init__(self, seed):
        super().__init__()
        torch.manual_seed(seed)
        self.body = nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.Conv2d(16, 16, 3, padding=1), nn.ReLU(),
                                  nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(16, 16))
        self.body.bfloat16().to(memory_format=torch.channels_last)
        self.gain = nn.Parameter(torch.ones(16))

    def forward(self, x):
        return self.body(x).float() * self.gain


def _model(kind):
    return (lambda seed: _Mlp(seed).cuda()) if kind == "mlp" else (lambda seed: _Conv(seed).cuda())


def _input(kind, r, step):
    g = torch.Generator(device="cuda").manual_seed(1000 * step + r)
    if kind == "mlp":
        return torch.randn(16, 33, device="cuda", generator=g).bfloat16()
    return torch.randn(4, 3, 8, 8, device="cuda", generator=g).bfloat16().contiguous(memory_format=torch.channels_last)


OPTS = {
    "sgd": (torch.optim.SGD, dict(lr=0.05, momentum=0.9, nesterov=True, fused=True)),
    "adam": (torch.optim.Adam, dict(lr=1e-3, fused=True)),
    "adamw": (torch.optim.AdamW, dict(lr=1e-3, fused=True)),
    "adamw_foreach": (torch.optim.AdamW, dict(lr=1e-3, foreach=True)),
}


def _groups(params, cls):
    params = list(params)
    first = {"params": [p for p in params if p.dim() > 1], "weight_decay": 0.1}
    if cls is not torch.optim.SGD:
        first["eps"] = 1e-6
    return [first, {"params": [p for p in params if p.dim() <= 1], "weight_decay": 0.0, "lr": 2e-3}]


class _HandHeld:
    """The reference: the unsharded mini-DDP's bf16 model with fp32 masters kept by hand."""

    def __init__(self, ddp, cls, kw):
        self.params = list(ddp.module.parameters())
        self.masters = [p.detach().float().clone() if p.dtype == torch.bfloat16 else p for p in self.params]
        groups = _groups(self.params, cls)
        idx = {id(p): i for i, p in enumerate(self.params)}
        self.opt = cls([dict(g, params=[self.masters[idx[id(p)]] for p in g["params"]]) for g in groups], **kw)

    def zero_grad(self):
        self.opt.zero_grad()
        for p in self.params:
            p.grad = None

    @torch.no_grad()
    def step(self):
        for p, m in zip(self.params, self.masters):
            if m is not p:
                m.grad = None if p.grad is None else p.grad.float()
        self.opt.step()
        for p, m in zip(self.params, self.masters):
            if m is not p:
                p.copy_(m)


def _load_kernels(W):
    """Every library kernel a W-rank run below launches, launched once on its own: a kernel's first launch (lazy module
    loading waits for the device) must not be issued behind a collective of rank 0 that the other ranks have not joined.
    The bf16 and fp32 (bf16 wire) buckets' reduce-scatters and twoshot allreduces, and both fused steps."""
    from tests import test_zero_gpu as ZG
    from tests import test_zero_overlap_gpu as ZO

    for mode in (N.B2_F32_WIRE_BF16, N.B2_BF16):
        ZG._check(W, mode, 4095, seed=1)
    ZO._check(W, N.B2_F32_WIRE_BF16, 4095, "sgd", seed=1, n_steps=1)
    _check(W, 4095, "sgd", seed=1, n_steps=1)


def _run(W, opt, kind, overlap, steps=4, zero_copy=True, accumulate=False, checkpoint_at=None):
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    torch.backends.cudnn.deterministic = True
    cls, kw = OPTS[opt]
    if overlap and kw.get("foreach"):
        pytest.skip("overlap_with_ddp runs its own fused step")
    algo = "twoshot" if W > 1 else "auto"  # one allreduce kernel per bucket mode, loaded by _load_kernels
    if W > 1:
        _load_kernels(W)
    ca, plain_ddps, sa = _ddps(W, _model(kind), algo=algo)
    cb, zero_ddps, sb = _ddps(W, _model(kind), zero_copy=zero_copy, algo=algo)

    def make(ds):
        return [ZeroRedundancyOptimizer(d, cls, params=_groups(d.module.parameters(), cls), overlap_with_ddp=overlap,
                                        master_weights=True, **kw) for d in ds]

    try:
        plain = [_HandHeld(d, cls, kw) for d in plain_ddps]
        zero = make(zero_ddps)
        for z, d in zip(zero, zero_ddps):  # each rank holds fp32 masters for its block of every bf16 bucket, nothing more
            bf = [b for b in d.buckets if b.dtype == torch.bfloat16]
            assert sum(m.numel() for m in z._master_flat.values()) == sum(b.block for b in bf)
            assert all(m.dtype == torch.float32 for m in z._master_flat.values()) and len(z._master_flat) == len(bf)
        sched_p = [torch.optim.lr_scheduler.StepLR(o.opt, step_size=2, gamma=0.5) for o in plain]
        sched_z = [torch.optim.lr_scheduler.StepLR(o, step_size=2, gamma=0.5) for o in zero]

        def loss(ddp, r, step):
            return ddp(_input(kind, r, step)).square().mean()

        def backward(r, step, ddp, o, s):
            with torch.cuda.stream(s):
                o.zero_grad()
                if accumulate:
                    with ddp.no_sync():
                        loss(ddp, r, step + 50).backward()
                loss(ddp, r, step).backward()

        def step_(o, sched, s):
            with torch.cuda.stream(s):
                o.step()
                sched.step()

        for ds, ss in ((plain_ddps, sa), (zero_ddps, sb)):
            for r, (d, s) in enumerate(zip(ds, ss)):
                with torch.cuda.stream(s), d.no_sync():
                    loss(d, r, 99).backward()
                d.module.zero_grad()
            torch.cuda.synchronize()
        for step in range(steps):
            if step == checkpoint_at:  # consolidate; fresh models and optimizers load the weights and the checkpoint
                _consolidate(zero, 0, sb)
                sd = zero[0].state_dict()
                weights = [d.module.state_dict() for d in zero_ddps]
                cc, zero_ddps, sb = _ddps(W, _model(kind), zero_copy=zero_copy, algo=algo)
                cb += cc
                for d, wts in zip(zero_ddps, weights):
                    d.module.load_state_dict(wts)
                zero = make(zero_ddps)
                for z in zero:
                    z.load_state_dict(sd)
                torch.cuda.synchronize()
                sched_z = [torch.optim.lr_scheduler.StepLR(o, step_size=2, gamma=0.5, last_epoch=step - 1) for o in zero]
                for o, p in zip(zero, plain):
                    for g, h in zip(o.param_groups, p.opt.param_groups):
                        g["lr"] = h["lr"]
            _phase(W, lambda r: backward(r, step, plain_ddps[r], plain[r], sa[r]))
            _phase(W, lambda r: backward(r, step, zero_ddps[r], zero[r], sb[r]))
            _phase(W, lambda r: step_(plain[r], sched_p[r], sa[r]))
            _phase(W, lambda r: step_(zero[r], sched_z[r], sb[r]))
            for r in range(W):
                for i, (a, b) in enumerate(zip(zero_ddps[r].module.parameters(), plain_ddps[r].module.parameters())):
                    _assert_bits(a, b, f"step {step} rank {r} param {i}")
        _consolidate(zero, 0, sb)
        sd = zero[0].state_dict()
        _assert_state_equal({k: sd[k] for k in ("state", "param_groups")}, plain[0].opt.state_dict(), "consolidated state")
        index = [p for g in _groups(plain[0].params, cls) for p in g["params"]]  # the optimizer's parameter order
        master_of = {id(p): m for p, m in zip(plain[0].params, plain[0].masters)}
        assert len(sd["master_params"]) == len(index)
        for i, (got, p) in enumerate(zip(sd["master_params"], index)):
            m = master_of[id(p)]
            if p.dtype == torch.float32:
                assert got is None, f"master {i}: an fp32 parameter has none"
            else:
                _assert_bits(got, m, f"master {i}")
        return zero_ddps, zero, sb
    finally:
        for c in ca + cb:
            c.close()


@pytest.mark.parametrize("overlap", [False, True], ids=["step", "overlap"])
@pytest.mark.parametrize("kind", ["mlp", "conv"])
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("W", [1, 2, 4])
def test_master_training_is_bit_equal_to_hand_held_masters(W, opt, kind, overlap):
    if W > 1:
        _run(1, opt, kind, overlap, steps=1)  # loads every compute kernel before the ranks wait on each other
    _run(W, opt, kind, overlap)


@pytest.mark.parametrize("overlap", [False, True], ids=["step", "overlap"])
def test_master_no_sync_accumulation_and_copy_in(overlap):
    _run(1, "adamw", "mlp", overlap, steps=1)
    _run(2, "adamw", "mlp", overlap, steps=3, accumulate=True)
    _run(2, "sgd", "conv", overlap, steps=3, zero_copy=False)


@pytest.mark.parametrize("overlap", [False, True], ids=["step", "overlap"])
def test_master_checkpoint_round_trip(overlap):
    _run(1, "adamw", "mlp", overlap, steps=1)
    _run(2, "adamw", "mlp", overlap, steps=4, checkpoint_at=2)
    _run(2, "sgd", "conv", overlap, steps=4, checkpoint_at=2)


def test_load_without_master_params_rederives_them_from_the_bf16_parameters():
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    comms, ddps, ss = _ddps(1, _model("mlp"))
    try:
        d, s = ddps[0], ss[0]
        z = ZeroRedundancyOptimizer(d, torch.optim.AdamW, master_weights=True, lr=1e-3)
        with torch.cuda.stream(s):
            d(_input("mlp", 0, 0)).square().mean().backward()
            z.step()
            z.consolidate_state_dict(0)
            sd = z.state_dict()
            assert len(sd["master_params"]) == len(list(d.module.parameters()))
            with torch.no_grad():
                for m in z._master_flat.values():
                    m.add_(1.0)  # stale masters
            z.load_state_dict({k: v for k, v in sd.items() if k != "master_params"})
        torch.cuda.synchronize()
        for bi, m in z._master_flat.items():
            b = d.buckets[bi]
            _assert_bits(m, b.param_flat[: b.block].float(), f"bucket {bi}")
    finally:
        for c in comms:
            c.close()


def test_split_parameter_without_overlap():
    """A block boundary that splits a parameter of a numel that is not a multiple of 4: refused for Adam(fused=True) with
    coupled weight decay, exact for AdamW(fused=True)."""
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    class _Odd(nn.Module):  # one bf16 parameter of 1001 elements, split between the two rank blocks; no GEMM
        def __init__(self):
            super().__init__()
            self.w = nn.Parameter(torch.randn(1001).bfloat16())

        def forward(self, x):
            return (x * self.w).float()

    def odd(seed):
        torch.manual_seed(seed)
        return _Odd().cuda()

    _load_kernels(2)
    comms, ddps, ss = _ddps(2, odd, algo="twoshot")
    try:
        with pytest.raises(ValueError, match="split between rank blocks"):
            ZeroRedundancyOptimizer(ddps[0], torch.optim.Adam, master_weights=True, lr=1e-3, weight_decay=0.1, fused=True)
    finally:
        for c in comms:
            c.close()
    ca, plain_ddps, sa = _ddps(2, odd, algo="twoshot")
    cb, zero_ddps, sb = _ddps(2, odd, algo="twoshot")
    try:
        kw = dict(lr=1e-3, weight_decay=0.1, fused=True)
        plain = [_HandHeld(d, torch.optim.AdamW, kw) for d in plain_ddps]
        for h in plain:  # one group: rebuild over every master
            h.opt = torch.optim.AdamW(h.masters, **kw)
        zero = [ZeroRedundancyOptimizer(d, torch.optim.AdamW, master_weights=True, **kw) for d in zero_ddps]
        B = zero_ddps[0].buckets
        assert any(o // b.block != (o + n - 1) // b.block and n % 4
                   for b in B for o, n in zip(b.spec.offsets, b.spec.numels)), "no parameter is split"
        def backward(d, o, s, r, step):
            with torch.cuda.stream(s):
                o.zero_grad()
                x = torch.randn(8, 1001, device="cuda", generator=torch.Generator(device="cuda").manual_seed(step * 10 + r))
                d(x.bfloat16()).float().square().mean().backward()

        def step_(o, s):
            with torch.cuda.stream(s):
                o.step()

        for step in range(3):
            for ds, os_, ss in ((plain_ddps, plain, sa), (zero_ddps, zero, sb)):
                _phase(2, lambda r: backward(ds[r], os_[r], ss[r], r, step))
                _phase(2, lambda r: step_(os_[r], ss[r]))
            for r in range(2):
                for i, (a, b) in enumerate(zip(zero_ddps[r].module.parameters(), plain_ddps[r].module.parameters())):
                    _assert_bits(a, b, f"step {step} rank {r} param {i}")
    finally:
        for c in ca + cb:
            c.close()


def test_master_run_time_errors():
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    comms, ddps, ss = _ddps(1, _model("mlp"))
    try:
        d, s = ddps[0], ss[0]
        z = ZeroRedundancyOptimizer(d, torch.optim.AdamW, master_weights=True, lr=1e-3)
        with torch.cuda.stream(s):
            d(_input("mlp", 0, 0)).square().mean().backward()
            with pytest.raises(RuntimeError, match="master_weights=True does not support GradScaler"):
                z.step(grad_scaler=torch.amp.GradScaler("cuda"))
            norm = z.clip_grad_norm_(1e-3)  # on the fp32 master gradients
            grads = [v.grad for v, _, _ in d._shard_grads if v.grad is not None]
            assert grads and all(g.dtype == torch.float32 for g in grads) and norm.dtype == torch.float32
            z.step()
        torch.cuda.synchronize()
    finally:
        for c in comms:
            c.close()
