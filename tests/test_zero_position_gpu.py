"""Where an element sits in its parameter, on the GPU: b2_reduce_scatter_step and ZeroRedundancyOptimizer wherever a rank's
block boundary splits a parameter.

torch's fused Adam with coupled weight decay rounds ``param * weight_decay`` by the element's index j in its parameter:
j % 4 on its vectorised path, (j % 65536) % 2048 / 512 on its scalar path (DESIGN.md 2.4).  So the fused step is checked
against torch._fused_adam_ / _fused_adamw_ / _fused_sgd_ applied to whole parameters, each its own tensor with its whole
reduced gradient and state, never to per-block slices; and each case is shown to be sensitive to position first: the same
launch with every run counted from index 0 (or with the other path's flag) must give other bits.  Then a model whose
parameters straddle block boundaries with a numel that is not a multiple of 4 trains bit-equal to the unsharded mini-DDP."""
import pytest
import torch

from tests.test_zero_gpu import (_assert_same, _assert_state_equal, _consolidate, _ddps, _input, _params, _phase, _warm,
                                 WIRE)
from tests.test_zero_overlap_gpu import _table, _world
from tests.test_zero_position import ODD_BIG, ODD_BOUNDARIES, _odd
from torchx_b200.ddp import _native as N
from torchx_b200.ddp import zero as Z

pytestmark = pytest.mark.gpu

# the positions a block boundary takes inside a parameter: both sides of the 512-element slots of the scalar path, of
# its 2048-element period and of the 65536-element chunks, and one past two chunks
PIDX = [1, 2, 3, 5, 511, 512, 513, 1535, 2047, 2048, 2049, 65535, 65536, 65537, 65536 + 1537, 131071]
TAIL = 65540  # elements of a straddling parameter past its boundary: a whole chunk, 32 periods of the scalar path
# Adam / AdamW with coupled or decoupled decay in both groups, maximize off (group 0) and on (group 1).  The gradients are of
# the size of param * weight_decay, so that their sum often cancels (whether the product was rounded on its own then shows
# even through a bf16 or fp16 wire, whose gradients have no bits below its ulp), and the state starts small against the
# update
ADAM = [dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.1, maximize=False),
        dict(lr=3e-3, beta1=0.8, beta2=0.99, eps=1e-6, weight_decay=0.05, maximize=True)]
SGD = [dict(lr=0.05, momentum=0.9, dampening=0.1, weight_decay=0.01, nesterov=False, maximize=False),
       dict(lr=0.02, momentum=0.8, dampening=0.0, weight_decay=0.0, nesterov=True, maximize=False)]
# kind -> (table kind, hyper-parameters, the group of the straddling parameters; the others take the other group)
KINDS = {"adam": ("adam", ADAM, 0), "adam_max": ("adam", ADAM, 1), "adamw": ("adamw", ADAM, 0), "sgd": ("sgd", SGD, 0)}
PATHS = ["vector", "scalar_numel", "scalar_align"]


def _sensitive(path, p):
    """Whether counting a run that starts at index p of its parameter from 0 instead changes the rounding of some element."""
    return p % 4 != 0 if path == "vector" else p % 2048 != 0


def _cases(W, path):
    """The pidx values of each bucket: one per block boundary (W - 1 of them), every bucket with at least one that is
    sensitive to position; at W = 2 the insensitive values make buckets of their own and are dropped."""
    sens = [p for p in PIDX if _sensitive(path, p)]
    insens = [p for p in PIDX if not _sensitive(path, p)] if W > 2 else []
    ordered = insens + sens
    nb = -(-len(ordered) // (W - 1))
    assert len(insens) <= nb <= len(sens)
    out = []
    for j in range(nb):
        ps = ordered[j::nb]
        out.append([ps[k % len(ps)] for k in range(W - 1)])
    return out


def _layout(W, pidx, path):
    """A bucket whose boundary k * B falls at index pidx[k - 1] of straddling parameter k (k = 1 .. W - 1), with fillers
    between them.  Returns B, n (3 elements short of W * B: a pad), and per parameter (offset, numel, straddles)."""
    def numel(k, p):  # the straddling parameter's numel: a multiple of 4 except on the scalar path by numel
        want = 0 if path != "scalar_numel" else 1 + k % 3
        return p + TAIL + (want - p - TAIL) % 4

    Ls = [numel(k, p) for k, p in enumerate(pidx)]
    B = (max(pidx) + max(L - p for L, p in zip(Ls, pidx)) + 40 + 7) // 8 * 8
    n = W * B - 3
    assert Z.padded_block(n, W) == B
    params, at = [], 0
    for k, (p, L) in enumerate(zip(pidx, Ls), start=1):
        o = k * B - p
        assert o > at
        params.append((at, o - at, False))
        params.append((o, L, True))
        at = o + L
    params.append((at, n - at, False))
    return B, n, params


def _ref_tensor(src, misaligned):
    """A whole parameter (or its gradient / state) as a tensor of its own: 1 element into its allocation when misaligned."""
    t = torch.empty(src.numel() + int(misaligned), device="cuda")[int(misaligned):]
    t.copy_(src)
    return t


def _torch_step(kind, hyper, gi, P, G, M, V, step):
    h = hyper[gi]
    if kind == "sgd":
        torch._fused_sgd_(P, G, M, weight_decay=h["weight_decay"], momentum=h["momentum"], lr=h["lr"],
                          dampening=h["dampening"], nesterov=h["nesterov"], maximize=h["maximize"], is_first_step=step == 0)
    else:
        fn = torch._fused_adam_ if kind == "adam" else torch._fused_adamw_
        steps = [torch.full((), float(step + 1), device="cuda") for _ in P]
        fn(P, G, M, V, [], steps, lr=h["lr"], beta1=h["beta1"], beta2=h["beta2"], weight_decay=h["weight_decay"],
           eps=h["eps"], amsgrad=False, maximize=h["maximize"])


def _sweep_bucket(W, mode, kind, path, pidx, seed, n_steps=3, stage_mb=8):
    """One bucket: the fused step on every rank's block against torch's fused optimizer on whole parameters, bit for bit
    after every step (parameters, both states, the pad untouched); the position-blind variants must differ (Adam with
    coupled decay, maximize off) or agree (the controls) after the first."""
    tkind, hyper, tgroup = KINDS[kind]
    w = _world(W, stage_mb)
    B, n, params = _layout(W, pidx, path)
    offsets = [o for o, _, _ in params]
    numels = [L for _, L, _ in params]
    groups = [tgroup if s else 1 - tgroup for *_, s in params]
    # the path torch's fused kernels take on each whole parameter: the scalar one for a numel that is not a multiple of 4
    # or (the straddling parameters of the misaligned case) a tensor that is not 16-byte aligned
    scalar = [L % 4 != 0 or (s and path == "scalar_align") for _, L, s in params]
    gen = torch.Generator().manual_seed(seed)
    full = [torch.randn(W * B, generator=gen).cuda(), torch.randn(W * B, generator=gen).cuda() * 0.01,
            torch.rand(W * B, generator=gen).cuda() * 1e-4]  # parameter, exp_avg / momentum, exp_avg_sq over the padded bucket
    blocks = [[t[r * B:(r + 1) * B].clone() for t in full] for r in range(W)]
    ref = [[_ref_tensor(t[o:o + L], scalar[i] and L % 4 == 0) if k == 0 else t[o:o + L].clone() for k, t in enumerate(full)]
           for i, (o, L, _) in enumerate(params)]
    tables, keep = [], []
    for r in range(W):
        x = torch.randn(n, generator=torch.Generator().manual_seed(seed * 10 + r)).cuda() * 0.1
        z = torch.zeros(W * B - n, device="cuda")
        keep += [x, z]
        segs = (N.B2Segment * 2)()
        segs[0].src, segs[0].begin, segs[0].end = x.data_ptr(), 0, n
        segs[1].src, segs[1].begin, segs[1].end = z.data_ptr(), n, W * B
        tables.append(segs)
    runs = [Z.block_runs(offsets, numels, groups, B, r) for r in range(W)]
    shards = [torch.empty(B, device="cuda") for _ in range(W)]
    wire = WIRE[mode]
    torch.cuda.synchronize()
    w.run(lambda r, c, s: c.reduce_scatter_gather_(shards[r], tables[r], 2, scale=1.0 / W, wire=wire, stream=s))
    grad = torch.cat(shards)
    grads = [_ref_tensor(grad[o:o + L], scalar[i] and L % 4 == 0) for i, (o, L, _) in enumerate(params)]

    def table(r, step, pos):
        rs = []
        for lo, hi, gi, i in runs[r]:
            if i is None:
                rs.append((lo, gi, 0.0))
            else:
                st = float(step == 0) if tkind == "sgd" else float(step + 1)
                rs.append((lo, gi, st, pos(i, lo + r * B - offsets[i], scalar[i])))
        return rs

    def launch(P, step, pos):
        opts = [_table(tkind, hyper, B, table(r, step, pos), *P[r]) for r in range(W)]
        w.run(lambda r, c, s: c.reduce_scatter_step_(B, tables[r], 2, opts[r], scale=1.0 / W, wire=wire, stream=s))

    def expected():
        out = [t.clone() for t in full]
        for (o, L, _), pr in zip(params, ref):
            for t, v in zip(out, pr):
                t[o:o + L] = v
        return out

    what = f"W={W} mode={mode} {kind} {path} pidx={pidx}"
    for step in range(n_steps):
        blind = []
        if step == 0:  # the same launch with the straddling parameters' runs counted from index 0, or on the other path
            straddles = [s for *_, s in params]
            for name, pos in (("index 0", lambda i, j, sc: (0 if straddles[i] else j, sc)),
                              ("other path", lambda i, j, sc: (j, sc != straddles[i]))):
                P = [[t.clone() for t in b] for b in blocks]
                launch(P, step, pos)
                blind.append((name, P))
        launch(blocks, step, lambda i, j, sc: (j, sc))
        for g in range(2):
            idx = [i for i in range(len(params)) if groups[i] == g]
            cols = list(zip(*[ref[i] for i in idx]))
            _torch_step(tkind, hyper, g, list(cols[0]), [grads[i] for i in idx], list(cols[1]), list(cols[2]), step)
        torch.cuda.synchronize()
        want = expected()
        for r in range(W):
            for name, got, t in zip(("param", "state0", "state1"), blocks[r], want):
                exp = t[r * B:(r + 1) * B]
                bad = (got.view(torch.int32) != exp.view(torch.int32)).nonzero().flatten()
                assert bad.numel() == 0, f"{what} step {step} rank {r} {name}: block elements {bad[:8].tolist()}"
        position_bound = tkind == "adam" and not hyper[tgroup]["maximize"]
        for name, P in blind:
            same = all(torch.equal(P[r][k].view(torch.int32), want[k][r * B:(r + 1) * B].view(torch.int32))
                       for r in range(W) for k in range(3))
            if position_bound:
                assert not same, f"{what}: the launch with {name} gives the same bits, so this case cannot fail"
            else:
                assert same, f"{what}: {kind} must not depend on where a run sits in its parameter ({name})"
    return B


MODES = {2: 1, 3: 3, 8: 0}  # the controls' mode at each world


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("mode", [0, 1, 3])
@pytest.mark.parametrize("W", [2, 3, 8])
def test_adam_coupled_decay_at_every_split_position(W, mode, path):
    for j, pidx in enumerate(_cases(W, path)):
        _sweep_bucket(W, mode, "adam", path, pidx, seed=W * 100 + mode * 10 + j)


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("kind", ["adam_max", "adamw", "sgd"])
@pytest.mark.parametrize("W", [2, 3, 8])
def test_position_independent_steps_at_every_split_position(W, kind, path):
    for j, pidx in enumerate(_cases(W, path)):
        _sweep_bucket(W, MODES[W], kind, path, pidx, seed=W * 100 + j, n_steps=1)


@pytest.mark.parametrize("path", ["scalar_numel", "scalar_align"])
def test_launch_boundary_inside_a_scalar_path_run(path):
    """stage_mb=1: the block is cut into launches, and the second launch (o.off != 0) starts inside the straddling
    parameter on rank 0, which torch steps on its scalar path."""
    W, mode, stage_mb, pidx = 2, 1, 1, [131071]
    B, n, params = _layout(W, pidx, path)
    cap = (((stage_mb << 20) // (W + 1)) & ~255) // 4  # fp32 wire: elements of a block one recv region holds
    o, L, _ = params[1]
    assert cap < B and o < cap < o + L and (cap - o) % 2048 >= 512  # a launch starts off slot 0 of the scalar path
    _sweep_bucket(W, mode, "adam", path, pidx, seed=77, stage_mb=stage_mb)


# ---- the mini-DDP on a model whose parameters straddle block boundaries ------------------------------------------------
def _groups(ddp, cls, wd):
    decay = [p for p in ddp.module.parameters() if p.dim() > 1]
    rest = [p for p in ddp.module.parameters() if p.dim() <= 1]
    first = {"params": decay, "weight_decay": wd[0]}
    if cls is not torch.optim.SGD:
        first["eps"] = 1e-6
    return [first, {"params": rest, "weight_decay": wd[1], "lr": 2e-3}]


# name -> (class, options of both the unsharded and the sharded optimizer, weight decay of the two groups)
ODD_OPTS = {
    "adamw_fused": (torch.optim.AdamW, dict(lr=1e-3, fused=True), (0.1, 0.01)),
    "sgd_fused": (torch.optim.SGD, dict(lr=0.05, momentum=0.9, nesterov=True, fused=True), (0.1, 0.01)),
    "adam_foreach": (torch.optim.Adam, dict(lr=1e-3, foreach=True), (0.1, 0.01)),
    "adam_max_fused": (torch.optim.Adam, dict(lr=1e-3, maximize=True, fused=True), (0.1, 0.01)),
    "sgd_max_foreach": (torch.optim.SGD, dict(lr=0.05, momentum=0.9, maximize=True, foreach=True), (0.0, 0.0)),
    "sgd_max_nomomentum_fused": (torch.optim.SGD, dict(lr=0.05, maximize=True, fused=True), (0.0, 0.0)),
    # refused by the sharded mode (a split parameter of a numel that is not a multiple of 4); the overlap mode steps Adam
    # exactly, and its fused SGD with maximize has the caveat of DESIGN.md 2.4, so that one is left out of overlap here
    "adam_fused": (torch.optim.Adam, dict(lr=1e-3, fused=True), (0.1, 0.01)),
    "sgd_max_fused": (torch.optim.SGD, dict(lr=0.05, momentum=0.9, maximize=True, fused=True), (0.0, 0.0)),
}


def _expected_positions(z, b):
    """(block begin, index in its parameter, scalar path) of every parameter run of this rank's block, from the layout."""
    r, B = z._rank, b.block
    out = []
    for o, n in zip(b.spec.offsets, b.spec.numels):
        lo, hi = max(o, r * B), min(o + n, (r + 1) * B)
        if lo < hi:
            out.append((lo - r * B, lo - o, n % 4 != 0))
    return out


def _train_odd(W, opt, overlap, steps=3):
    from torchx_b200.ddp import ZeroRedundancyOptimizer

    cls, kw, wd = ODD_OPTS[opt]
    ca, plain_ddps, sa = _ddps(W, _odd)
    cb, zero_ddps, sb = _ddps(W, _odd)
    try:
        plain = [cls(_groups(d, cls, wd), **kw) for d in plain_ddps]
        zero = [ZeroRedundancyOptimizer(d, cls, params=_groups(d, cls, wd), overlap_with_ddp=overlap, **kw)
                for d in zero_ddps]
        if overlap:  # the positions the host hands the kernel, against the layout
            big = set()  # where the big weight's runs start in it, over all ranks
            for z in zero:
                for b in z.model.buckets:
                    t = z._launch_table(b)
                    got = [(t.run_begin[k], t.run_index[k], bool(t.run_scalar[k])) for k in range(t.n_runs)
                           if t.run_group[k] != N.B2_OPT_NO_GROUP]
                    if cls is torch.optim.Adam:
                        assert got == _expected_positions(z, b), (W, z._rank, b.spec.index, got)
                        if ODD_BIG in b.spec.numels:
                            big |= {j for _, j, s in got if s}
                    else:
                        assert all(j == 0 and not s for _, j, s in got), got  # position-independent: never marked
            if cls is torch.optim.Adam:
                assert sorted(big) == [0] + ODD_BOUNDARIES[W], big
        _warm(plain_ddps, sa, "mlp")
        _warm(zero_ddps, sb, "mlp")

        def backward(r, step, ddp, o, s):
            with torch.cuda.stream(s):
                o.zero_grad()
                ddp(_input("mlp", r, step)).square().mean().backward()

        def step_(o, s):
            with torch.cuda.stream(s):
                o.step()

        for step in range(steps):
            _phase(W, lambda r: backward(r, step, plain_ddps[r], plain[r], sa[r]))
            _phase(W, lambda r: backward(r, step, zero_ddps[r], zero[r], sb[r]))
            _phase(W, lambda r: step_(plain[r], sa[r]))
            _phase(W, lambda r: step_(zero[r], sb[r]))
            for r in range(W):
                _assert_same(_params(zero_ddps[r]), _params(plain_ddps[r]), f"{opt} overlap={overlap} W={W} step {step} rank {r}")
        _consolidate(zero, 0, sb)
        _assert_state_equal(zero[0].state_dict(), plain[0].state_dict(), f"{opt} overlap={overlap} W={W} consolidated")
    finally:
        for c in ca + cb:
            c.close()


@pytest.mark.parametrize("opt", ["adam_fused", "adamw_fused", "sgd_fused"])
@pytest.mark.parametrize("W", [2, 3, 4])
def test_odd_model_overlap_is_bit_equal_to_fused_unsharded(W, opt):
    _train_odd(1, opt, True, steps=1)  # loads every compute kernel before the ranks wait on each other
    _train_odd(W, opt, True)


@pytest.mark.parametrize("opt", ["adam_foreach", "adamw_fused", "sgd_fused", "adam_max_fused", "sgd_max_foreach",
                                 "sgd_max_nomomentum_fused"])
@pytest.mark.parametrize("W", [2, 3, 4])
def test_odd_model_sharded_is_bit_equal_to_unsharded(W, opt):
    _train_odd(1, opt, False, steps=1)
    _train_odd(W, opt, False)


@pytest.mark.parametrize("opt", ["adam_fused", "sgd_max_fused"])
@pytest.mark.parametrize("W", [2, 3, 4])
def test_odd_model_sharded_refuses_fused_steps_that_depend_on_the_split(W, opt):
    with pytest.raises(ValueError, match=r"parameter '4\.weight' \(131455 elements"):
        _train_odd(W, opt, False)
    _train_odd(1, opt, False, steps=2)  # one block: nothing is split, and the same options train bit-equal


@pytest.mark.parametrize("W", [2, 3, 4])
def test_refused_fused_steps_do_differ_on_block_views(W):
    """Why the sharded mode refuses them: stepping the rank-block views of the big weight with torch's fused Adam with
    coupled decay, or its fused SGD with maximize, momentum and no decay, gives other bits than stepping it whole."""
    B = Z.padded_block(ODD_BIG, W)
    gen = torch.Generator().manual_seed(W)
    p, g, m = (torch.randn(ODD_BIG, generator=gen).cuda() for _ in range(3))
    v = torch.rand(ODD_BIG, generator=gen).cuda()
    views = [slice(r * B, min((r + 1) * B, ODD_BIG)) for r in range(W)]
    for kind, hyper, gi in (("adam", ADAM, 0), ("sgd", [dict(lr=0.05, momentum=0.9, dampening=0.0, weight_decay=0.0,
                                                              nesterov=False, maximize=True)], 0)):
        whole = [t.clone() for t in (p, m, v)]
        piece = [t.clone() for t in (p, m, v)]
        for step in range(2):  # the fused SGD's first step only copies the gradient into the momentum buffer
            _torch_step(kind, hyper, gi, [whole[0]], [g], [whole[1]], [whole[2]], step)
            _torch_step(kind, hyper, gi, [piece[0][s] for s in views], [g[s] for s in views], [piece[1][s] for s in views],
                        [piece[2][s] for s in views], step)
        torch.cuda.synchronize()
        assert not all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(whole, piece)), (W, kind)
