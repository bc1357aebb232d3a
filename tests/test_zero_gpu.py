"""b2_reduce_scatter_gather and the ZeRO-1 mini-DDP on the GPU, all ranks sharing one device.

Kernel: rank r's shard against the oracles (oracle.allreduce for modes 0-2, tests/oracle_f16.c for modes 3-4) and against
allreduce_gather_ of the same table on the same communicator, block for block and bit for bit, in all five modes at
W = 1, 2, 3, 4, 8; ragged sizes, parameter boundaries inside and across blocks, the zero pad, the one-segment table, and
blocks larger than a stage region.  Mini-DDP: ZeroRedundancyOptimizer against the unsharded mini-DDP with the plain
optimizer, bit for bit after every step; GradScaler, no_sync, clip_grad_norm_ and checkpoints."""
import threading

import numpy as np
import pytest
import torch
from torch import nn

import oracle
from tests import _oracle_f16 as F16
from tests._util import World, assert_bits_equal
from torchx_b200.ddp import _native as N
from torchx_b200.ddp.zero import padded_block

pytestmark = pytest.mark.gpu

WIRE = {N.B2_F32_WIRE_BF16: "bf16", N.B2_F32: "f32", N.B2_BF16: "bf16", N.B2_F32_WIRE_F16: "f16", N.B2_F16: "f16"}
DTYPE = {N.B2_F32_WIRE_BF16: torch.float32, N.B2_F32: torch.float32, N.B2_BF16: torch.bfloat16,
         N.B2_F32_WIRE_F16: torch.float32, N.B2_F16: torch.float16}
_WORLDS = {}


def _world(W, stage_mb=8):
    key = (W, stage_mb)
    if key not in _WORLDS:
        _WORLDS[key] = World([0] * W, stage_mb=stage_mb, timeout_s=20.0)
        for c in _WORLDS[key].comms:
            c.set_max_ctas(max(1, 32 // W))  # every rank's kernels co-resident on the one device with room to spare
    return _WORLDS[key]


@pytest.fixture(scope="module", autouse=True)
def _close_worlds():
    yield
    for w in _WORLDS.values():
        w.close()
    _WORLDS.clear()


def _host(t):
    """A device bucket as the oracles take it: fp32 values, or the 16-bit patterns."""
    t = t.detach().cpu()
    if t.dtype == torch.float32:
        return t.numpy()
    return t.view(torch.int16).numpy().view(np.uint16)


def _oracle(mode, xs, scale):
    if mode in (N.B2_F32_WIRE_F16, N.B2_F16):
        return F16.allreduce(mode, xs, scale)
    return oracle.allreduce(mode, xs, scale)


def _pieces(n, rng, one_segment):
    """Parameter sizes that cover n elements: a mix of tiny and large ones, so that boundaries fall inside and across
    blocks and on and off vecs."""
    if one_segment:
        return [n]
    sizes, left = [], n
    while left:
        k = int(min(left, rng.choice([1, 3, 8, 13, 100, 1000, 40000])))
        sizes.append(k)
        left -= k
        if len(sizes) == N.B2_MAX_SEGMENTS - 2:
            sizes.append(left)
            break
    return [s for s in sizes if s]


def _check(W, mode, n, seed, one_segment=False, stage_mb=8):
    w = _world(W, stage_mb)
    dt = DTYPE[mode]
    B = padded_block(n, W)
    rng = np.random.default_rng(seed)
    sizes = _pieces(n, rng, one_segment)
    xs, tables, keep = [], [], []
    for r in range(W):
        x = torch.randn(n, generator=torch.Generator().manual_seed(seed * 10 + r)).to(dt).cuda()
        xs.append(x)
        # every parameter its own allocation, every other one off a vec (element offset 1)
        segs = (N.B2Segment * (len(sizes) + 1))()
        at = 0
        for i, k in enumerate(sizes):
            t = torch.empty(k + (i % 2), dtype=dt, device="cuda")[i % 2:]
            t.copy_(x[at:at + k])
            keep.append(t)
            segs[i].src, segs[i].begin, segs[i].end = t.data_ptr(), at, at + k
            at += k
        nseg = len(sizes)
        if W * B > n:
            z = torch.zeros(W * B - n, dtype=dt, device="cuda")
            keep.append(z)
            segs[nseg].src, segs[nseg].begin, segs[nseg].end = z.data_ptr(), n, W * B
            nseg += 1
        tables.append((segs, nseg))
    shards = [torch.full((B,), float("nan"), dtype=dt, device="cuda") for _ in range(W)]
    wire = WIRE[mode]
    torch.cuda.synchronize()  # the inputs are written on this thread's stream, the ranks run on their own
    w.run(lambda r, c, s: c.reduce_scatter_gather_(shards[r], tables[r][0], tables[r][1], scale=1.0 / W, wire=wire, stream=s))
    # the unsharded bucket allreduce of the same gradients (without the pad) on the same communicator
    buckets = [torch.empty(n, dtype=dt, device="cuda") for _ in range(W)]
    # one algorithm for every launch: a kernel's first launch (lazy module loading) must not wait behind rank 0's others
    w.run(lambda r, c, s: c.allreduce_gather_(buckets[r], tables[r][0], len(sizes), scale=1.0 / W, wire=wire,
                                              algo="twoshot" if W > 1 else "auto", stream=s))
    want = _oracle(mode, [_host(x) for x in xs], 1.0 / W)
    what = f"W={W} mode={mode} n={n} segs={len(sizes)}"
    for r in range(W):
        got = _host(shards[r])
        lo, hi = r * B, min((r + 1) * B, n)
        k = max(hi - lo, 0)
        assert_bits_equal(got[:k], _host(buckets[r])[lo:hi], f"{what} rank {r} vs allreduce_gather_")
        assert_bits_equal(got[:k], want[lo:hi], f"{what} rank {r} vs oracle")
        assert not got[k:].any(), f"{what} rank {r}: the pad must reduce to +0"


@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("W", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("n", [1, 7, 9, 4095, (1 << 17) + 3])
def test_reduce_scatter_gather_matches_oracle_and_allreduce(W, mode, n):
    _check(W, mode, n, seed=n % 97 + W)


@pytest.mark.parametrize("W,mode", [(2, 0), (3, 3), (4, 1), (8, 2)])
def test_reduce_scatter_gather_one_segment(W, mode):
    _check(W, mode, 50_001, seed=5, one_segment=True)


@pytest.mark.parametrize("W,mode", [(2, 1), (2, 0), (4, 4)])
def test_reduce_scatter_gather_block_larger_than_a_stage_region(W, mode):
    # stage_mb=8: a region holds 8 MiB / (W + 1) of wire data, far less than one block here - several launches
    n = 6_000_003
    assert padded_block(n, W) * (4 if mode == 1 else 2) > (8 << 20) // (W + 1)
    _check(W, mode, n, seed=11, stage_mb=8)


def test_reduce_scatter_gather_validates_its_table():
    w = _world(2)
    c = w.comms[0]
    out = torch.zeros(8, device="cuda")
    segs = (N.B2Segment * 1)()
    segs[0].src, segs[0].begin, segs[0].end = out.data_ptr(), 0, 15
    L = N.lib()
    assert L.b2_reduce_scatter_gather(c._h, out.data_ptr(), 8, segs, 1, 1, 1.0, None) == N.B2_EINVAL
    assert b"b2_reduce_scatter_gather: segments cover 15 elements, bucket has 16" in L.b2_last_error()
    assert L.b2_reduce_scatter_gather(c._h, out.data_ptr(), 8, segs, 0, 1, 1.0, None) == N.B2_EINVAL
    assert b"b2_reduce_scatter_gather: need 1..128 segments (got 0)" in L.b2_last_error()
    segs[0].begin = 1
    assert L.b2_reduce_scatter_gather(c._h, out.data_ptr(), 8, segs, 1, 1, 1.0, None) == N.B2_EINVAL
    assert b"b2_reduce_scatter_gather: segment 0 does not continue the bucket at element 0" in L.b2_last_error()
    assert L.b2_reduce_scatter_gather(c._h, None, 8, segs, 1, 1, 1.0, None) == N.B2_EINVAL
    assert b"b2_reduce_scatter_gather: null buffer" in L.b2_last_error()


# ---- the sharded mini-DDP -------------------------------------------------------------------------------------------
# Every parameter size is a multiple of 16 elements, so every parameter of the flat buffer starts 64-byte aligned, as in
# its own allocation: cuBLAS / cuDNN pick kernels by pointer alignment, and the bit-for-bit comparison needs the same ones.
def _mlp(seed):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(33, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 16)).cuda()


def _conv(seed):
    torch.manual_seed(seed)
    m = nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.BatchNorm2d(16), nn.ReLU(), nn.Conv2d(16, 16, 3, padding=1),
                      nn.BatchNorm2d(16), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(16, 16))
    return m.cuda().to(memory_format=torch.channels_last)


def _input(kind, r, step):
    g = torch.Generator(device="cuda").manual_seed(1000 * step + r)
    if kind == "mlp":
        return torch.randn(16, 33, device="cuda", generator=g)
    return torch.randn(4, 3, 8, 8, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)


def _phase(W, fn):
    """fn(rank) for every rank from this thread, then a device sync.  A step is cut into such phases (backward, optimizer
    step, ...) so that the first launch of a kernel (lazy module loading waits for the device) never waits behind a
    collective of rank 0 whose peers this thread has not issued yet."""
    for r in range(W):
        fn(r)
    torch.cuda.synchronize()


def _warm(ddps, streams, kind):
    """One local (no_sync) forward and backward per rank on its stream: loads every compute kernel the ranks' backwards
    will run while no collective is in flight."""
    for r, (d, s) in enumerate(zip(ddps, streams)):
        with torch.cuda.stream(s), d.no_sync():
            d(_input(kind, r, 99)).square().mean().backward()
    torch.cuda.synchronize()


def _threads(W, fn):
    """One host thread per rank: a host sync inside one rank (GradScaler, state_dict) must not stop the others."""
    errs = []

    def body(r):
        try:
            fn(r)
        except BaseException as e:  # noqa: BLE001
            errs.append((r, e))

    ts = [threading.Thread(target=body, args=(r,)) for r in range(W)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0][1]


def _consolidate(zero, to, streams):
    """consolidate_state_dict on every rank (each on its own stream), rank `to` last: only its call waits for the
    gathered state on the host."""
    for r in [q for q in range(len(zero)) if q != to] + [to]:
        with torch.cuda.stream(streams[r]):
            zero[r].consolidate_state_dict(to=to)
    torch.cuda.synchronize()
    for z in zero:
        z.comm.check()


def _ddps(W, model, wire="bf16", **kw):
    """W ranks of a mini-DDP on one device, constructed together (the constructor broadcasts rank 0's parameters)."""
    from torchx_b200.ddp import Communicator, DistributedDataParallel

    # the constructor's broadcast runs per dtype with a cat / copy between: load those kernels first (lazy module loading
    # waits for the device, where rank 0's first broadcast would be waiting for rank 1's)
    m = model(0)
    for dt in {t.dtype for t in [*m.parameters(), *m.buffers()]}:
        ts = [t.detach() for t in [*m.parameters(), *m.buffers()] if t.dtype == dt]
        flat = torch.cat([t.reshape(-1) for t in ts])
        torch._foreach_copy_(ts, [o.view_as(t) for o, t in zip(torch.split(flat, [t.numel() for t in ts]), ts)])
    torch.cuda.synchronize()
    comms = Communicator.create_local([0] * W, stage_mb=8)
    for c in comms:
        c.set_timeout(20.0)
        c.set_max_ctas(max(1, 64 // W))
    streams = [torch.cuda.Stream() for _ in range(W)]
    ddps = []
    for r in range(W):
        with torch.cuda.stream(streams[r]):
            ddps.append(DistributedDataParallel(model(r), comms[r], wire=wire, bucket_cap_mb=0.01, first_bucket_mb=0.004,
                                                broadcast_buffers=False, **kw))
    torch.cuda.synchronize()
    return comms, ddps, streams


def _groups(ddp):
    decay = [p for n, p in ddp.module.named_parameters() if p.dim() > 1]
    rest = [p for n, p in ddp.module.named_parameters() if p.dim() <= 1]
    return [{"params": decay, "weight_decay": 0.1}, {"params": rest, "weight_decay": 0.0, "lr": 2e-3}]


OPTS = {
    "sgd": (torch.optim.SGD, dict(lr=0.05, momentum=0.9)),
    "adam": (torch.optim.Adam, dict(lr=1e-3)),
    "adamw_foreach": (torch.optim.AdamW, dict(lr=1e-3, foreach=True)),
    "adamw_fused": (torch.optim.AdamW, dict(lr=1e-3, fused=True)),
}


def _params(ddp):
    return [p.detach().clone() for p in ddp.module.parameters()]


def _assert_same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and torch.equal(x.contiguous().view(torch.int32), y.contiguous().view(torch.int32)), f"{what} param {i}"


def _assert_state_equal(sd_a, sd_b, what):
    assert sd_a["param_groups"] == sd_b["param_groups"], what
    assert sorted(sd_a["state"]) == sorted(sd_b["state"]), what
    for i in sd_a["state"]:
        sa, sb = sd_a["state"][i], sd_b["state"][i]
        assert list(sa) == list(sb), (what, i)
        for k in sa:
            x, y = sa[k].cpu(), sb[k].cpu()
            bad = (x != y).nonzero().tolist() if x.shape == y.shape else "shape"
            assert torch.equal(x, y), (what, i, k, x.shape, bad[:8], len(bad), (x - y).abs().max().item())


@pytest.mark.parametrize("kind", ["mlp", "conv"])
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("W", [2, 4])
def test_sharded_training_is_bit_equal_to_unsharded(W, opt, kind):
    # W = 1 first: every compute kernel of the procedure is loaded before the ranks wait on each other (lazy module
    # loading waits for the device)
    _train_and_compare(1, opt, kind)
    _train_and_compare(W, opt, kind)


def _train_and_compare(W, opt, kind):
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    torch.backends.cudnn.deterministic = True
    cls, kw = OPTS[opt]
    model = _mlp if kind == "mlp" else _conv
    ca, plain_ddps, sa = _ddps(W, model)
    cb, zero_ddps, sb = _ddps(W, model)
    try:
        assert len(zero_ddps[0].buckets) >= 2 or W == 1
        plain = [cls(_groups(d), **kw) for d in plain_ddps]
        zero = [ZeroRedundancyOptimizer(d, cls, params=_groups(d), **kw) for d in zero_ddps]
        sched_p = [torch.optim.lr_scheduler.StepLR(o, step_size=2, gamma=0.5) for o in plain]
        sched_z = [torch.optim.lr_scheduler.StepLR(o, step_size=2, gamma=0.5) for o in zero]
        assert zero_ddps[0].buckets[0].flat is None  # the full-size gradient bucket is not kept

        def backward(r, step, ddp, opt, s):
            with torch.cuda.stream(s):
                opt.zero_grad()
                ddp(_input(kind, r, step)).square().mean().backward()

        def step_(opt, sched, s):
            with torch.cuda.stream(s):
                opt.step()
                sched.step()

        _warm(plain_ddps, sa, kind)
        _warm(zero_ddps, sb, kind)
        for step in range(4):
            _phase(W, lambda r: backward(r, step, plain_ddps[r], plain[r], sa[r]))
            _phase(W, lambda r: backward(r, step, zero_ddps[r], zero[r], sb[r]))
            assert all(p.grad is None for d in zero_ddps for p in d.module.parameters())
            _phase(W, lambda r: step_(plain[r], sched_p[r], sa[r]))
            _phase(W, lambda r: step_(zero[r], sched_z[r], sb[r]))
            for r in range(W):
                _assert_same(_params(zero_ddps[r]), _params(plain_ddps[r]), f"step {step} rank {r}")
                assert zero[r].param_groups[0]["lr"] == plain[r].param_groups[0]["lr"]
        _consolidate(zero, 0, sb)
        _assert_state_equal(zero[0].state_dict(), plain[0].state_dict(), "consolidated state")
    finally:
        for c in ca + cb:
            c.close()


def test_checkpoint_round_trip_and_clip_grad_norm():
    _checkpoint_and_clip(1)  # loads every compute kernel first, as above
    _checkpoint_and_clip(2)


def _checkpoint_and_clip(W):
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    ca, plain_ddps, sa = _ddps(W, _mlp)
    cb, zero_ddps, sb = _ddps(W, _mlp)
    try:
        plain = [torch.optim.AdamW(d.parameters(), lr=1e-3) for d in plain_ddps]
        zero = [ZeroRedundancyOptimizer(d, torch.optim.AdamW, lr=1e-3) for d in zero_ddps]
        norms = [None] * W

        def run(step, clip):
            for ddps, opts, ss in ((plain_ddps, plain, sa), (zero_ddps, zero, sb)):
                def bwd(r):
                    with torch.cuda.stream(ss[r]):
                        opts[r].zero_grad()
                        ddps[r](_input("mlp", r, step)).square().mean().backward()
                _phase(W, bwd)
            if clip:
                def clip_plain(r):
                    with torch.cuda.stream(sa[r]):
                        norms[r] = (torch.nn.utils.clip_grad_norm_(plain_ddps[r].parameters(), 1e-3),)

                def clip_zero(r):
                    with torch.cuda.stream(sb[r]):
                        norms[r] += (zero[r].clip_grad_norm_(1e-3),)
                _phase(W, clip_plain)
                _phase(W, clip_zero)
            for opts, ss in ((plain, sa), (zero, sb)):
                def stp(r):
                    with torch.cuda.stream(ss[r]):
                        opts[r].step()
                _phase(W, stp)

        _warm(plain_ddps, sa, "mlp")
        _warm(zero_ddps, sb, "mlp")
        run(0, False)
        run(1, True)
        assert all(torch.equal(norms[0][1], n[1]) for n in norms)  # the same bits on every rank
        torch.testing.assert_close(norms[0][1], norms[0][0], rtol=1e-5, atol=0)
        assert norms[0][1] > 1e-3  # it did clip
        # sharded -> full state dict -> a plain AdamW over the unsharded mini-DDP, and back
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        _consolidate(zero, 0, sb)
        # the consolidated state lives in host memory on rank 0 only; no rank keeps anything on the GPU
        assert torch.cuda.memory_allocated() == before
        for r in range(1, W):
            with pytest.raises(RuntimeError, match="on rank `to` only"):
                zero[r].state_dict()
        full = zero[0].state_dict()
        assert all(not t.is_cuda for st in full["state"].values() for t in st.values())
        _assert_state_equal(full, plain[0].state_dict(), "consolidated")
        fresh = torch.optim.AdamW(plain_ddps[0].parameters(), lr=1e-3)
        fresh.load_state_dict(full)
        _assert_state_equal(fresh.state_dict(), full, "plain after load")
        for r in range(W):
            zero[r].load_state_dict(plain[0].state_dict())
        _consolidate(zero, W - 1, sb)
        _assert_state_equal(zero[W - 1].state_dict(), plain[0].state_dict(), "sharded after load")
        run(2, False)
        for r in range(W):
            _assert_same(_params(zero_ddps[r]), _params(plain_ddps[r]), f"after reload rank {r}")
    finally:
        for c in ca + cb:
            c.close()


def test_grad_scaler_skips_on_every_rank_and_no_sync():
    _scaler(1)  # loads every compute kernel first, as above
    _scaler(2)


def _scaler(W):
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    cb, ddps, sb = _ddps(W, _mlp, wire="f16")
    try:
        zero = [ZeroRedundancyOptimizer(d, torch.optim.AdamW, lr=1e-3) for d in ddps]
        scalers = [torch.amp.GradScaler("cuda", init_scale=2.0 ** 12) for _ in range(W)]

        def run(r, step, plant):
            x = _input("mlp", r, step)
            with torch.cuda.stream(sb[r]):
                zero[r].zero_grad()
                with ddps[r].no_sync():  # accumulation step: local gradients only
                    with torch.autocast("cuda", dtype=torch.float16):
                        scalers[r].scale(ddps[r](x).square().mean()).backward()
                with torch.autocast("cuda", dtype=torch.float16):
                    scalers[r].scale(ddps[r](x + 1).square().mean()).backward()
                if plant and r == W - 1:
                    ddps[r].buckets[0].shard_grad[3] = float("inf")  # the last rank's shard only
                scalers[r].step(zero[r])
                scalers[r].update()

        # each collective kind of the step once, one synchronised phase each, before the ranks run on their own threads
        _phase(W, lambda r: cb[r].allreduce_op_(torch.zeros((), device="cuda"), "max", stream=sb[r]))
        _phase(W, lambda r: cb[r].allgather_(torch.zeros(2 * W, device="cuda"), torch.zeros(2, device="cuda"), stream=sb[r]))
        before = [_params(d) for d in ddps]
        _threads(W, lambda r: run(r, 0, True))
        torch.cuda.synchronize()
        for r in range(W):
            _assert_same(_params(ddps[r]), before[r], f"rank {r} must have skipped the step")
            assert scalers[r].get_scale() == 2.0 ** 11
        _threads(W, lambda r: run(r, 1, False))
        torch.cuda.synchronize()
        assert all(sc.get_scale() == 2.0 ** 11 for sc in scalers)
        _assert_same(_params(ddps[0]), _params(ddps[-1]), "ranks agree")
        assert not all(torch.equal(a, b) for a, b in zip(_params(ddps[0]), before[0])), "the second step must have stepped"
    finally:
        for c in cb:
            c.close()


def test_no_sync_accumulation_matches_unsharded():
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    W = 2
    ca, plain_ddps, sa = _ddps(W, _mlp)
    cb, zero_ddps, sb = _ddps(W, _mlp)
    try:
        plain = [torch.optim.SGD(d.parameters(), lr=0.1, momentum=0.9) for d in plain_ddps]
        zero = [ZeroRedundancyOptimizer(d, torch.optim.SGD, lr=0.1, momentum=0.9) for d in zero_ddps]

        def bwd(r, step, ddp, opt, s):
            with torch.cuda.stream(s):
                opt.zero_grad()
                with ddp.no_sync():
                    ddp(_input("mlp", r, step)).sum().backward()
                ddp(_input("mlp", r, step + 50)).sum().backward()

        def stp(opt, s):
            with torch.cuda.stream(s):
                opt.step()

        for step in range(2):
            _phase(W, lambda r: bwd(r, step, plain_ddps[r], plain[r], sa[r]))
            _phase(W, lambda r: bwd(r, step, zero_ddps[r], zero[r], sb[r]))
            _phase(W, lambda r: stp(plain[r], sa[r]))
            _phase(W, lambda r: stp(zero[r], sb[r]))
            for r in range(W):
                _assert_same(_params(zero_ddps[r]), _params(plain_ddps[r]), f"step {step} rank {r}")
    finally:
        for c in ca + cb:
            c.close()


def test_sharding_after_a_backward_raises():
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    cb, ddps, sb = _ddps(1, _mlp)
    try:
        ddps[0](_input("mlp", 0, 0)).sum().backward()
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match="before the model's first backward"):
            ZeroRedundancyOptimizer(ddps[0], torch.optim.SGD, lr=0.1)
    finally:
        for c in cb:
            c.close()


def test_second_synced_backward_before_zero_grad_raises():
    """Unsharded, a second synced backward adds into the reduced gradients; sharded they live only in the shards, which it
    would overwrite, so it raises before launching anything, and works again after zero_grad()."""
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    for W in (1, 2):
        cb, ddps, sb = _ddps(W, _mlp)
        try:
            zero = [ZeroRedundancyOptimizer(d, torch.optim.SGD, lr=0.1) for d in ddps]
            _warm(ddps, sb, "mlp")

            def bwd(r, step):
                with torch.cuda.stream(sb[r]):
                    ddps[r](_input("mlp", r, step)).sum().backward()

            for z in zero:
                z.zero_grad()
            _phase(W, lambda r: bwd(r, 0))
            for r in range(W):
                with pytest.raises(RuntimeError, match="second synced backward before zero_grad"):
                    bwd(r, 1)
            torch.cuda.synchronize()
            def stp(r):
                with torch.cuda.stream(sb[r]):
                    zero[r].step()

            _phase(W, stp)
            for z in zero:
                z.zero_grad()
            _phase(W, lambda r: bwd(r, 2))  # after zero_grad() a synced backward runs again
            for c in cb:
                c.check()
        finally:
            for c in cb:
                c.close()


class _WithScalar(nn.Module):
    def __init__(self, seed):
        super().__init__()
        self.mlp = _mlp(seed)
        self.gain = nn.Parameter(torch.tensor(1.5, device="cuda"))  # a 0-dim parameter

    def forward(self, x):
        return self.mlp(x) * self.gain


def test_checkpoint_with_a_zero_dim_parameter():
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    cb, ddps, sb = _ddps(1, _WithScalar)
    try:
        zero = ZeroRedundancyOptimizer(ddps[0], torch.optim.AdamW, lr=1e-3)
        with torch.cuda.stream(sb[0]):
            zero.zero_grad()
            ddps[0](_input("mlp", 0, 0)).square().mean().backward()
            zero.step()
        _consolidate([zero], 0, sb)
        full = zero.state_dict()
        i = [p for ps in zero._full_groups for p in ps].index(ddps[0].module.gain)
        assert full["state"][i]["exp_avg"].shape == ()
        zero.load_state_dict(full)
        _consolidate([zero], 0, sb)
        _assert_state_equal(zero.state_dict(), full, "0-dim parameter after load")
    finally:
        for c in cb:
            c.close()
