"""ZeRO stage 1 for the mini-DDP: each rank keeps the optimizer state of one block of every bucket (DESIGN.md 2.5).

torch's ``ZeroRedundancyOptimizer`` needs a ``torch.distributed`` process group; under ``init_pg("b200")`` there is none.
This one runs on the native communicator instead:

  * the backward reduce-scatters every bucket into this rank's gradient shard (``b2_reduce_scatter_gather``: the bits the
    unsharded bucket allreduce leaves in that block, read zero-copy from the per-parameter gradients);
  * ``step()`` steps the inner optimizer on this rank's slice of the parameters only, then all-gathers every bucket's
    flat parameter buffer in place (exact bytes).

SGD, Adam and AdamW are elementwise, so stepping a slice gives the bits of stepping the whole tensor, with two exceptions
in torch's fused kernels (DESIGN.md 2.4) that the constructor refuses where they would apply: the parameters stay
bit-equal to those of the unsharded mini-DDP under the same optimizer, and the consolidated state to its state.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch

from . import _native as N
from .ddp import DistributedDataParallel, _view_like

# the elementwise optimizers: a slice of a tensor steps to the bits of the same slice of the stepped tensor (two fused
# exceptions: _check_split_params)
SUPPORTED = (torch.optim.SGD, torch.optim.Adam, torch.optim.AdamW)


def padded_block(numel: int, world: int) -> int:
    """Elements of one rank's block of a bucket of ``numel`` elements: ceil(numel / world) rounded up to a whole vec
    (8 elements), so every block starts on a vec.  The bucket is padded to world * block elements."""
    return (-(-numel // world) + 7) // 8 * 8


def block_intersections(offsets: Sequence[int], numels: Sequence[int], block: int, rank: int) -> List[Tuple[int, int, int]]:
    """(index, lo, hi) for each parameter whose bucket range [offset, offset + numel) meets rank's block
    [rank * block, (rank + 1) * block): bucket elements [lo, hi) of parameter ``index`` belong to this rank."""
    b0, b1 = rank * block, (rank + 1) * block
    out = []
    for i, (o, n) in enumerate(zip(offsets, numels)):
        lo, hi = max(o, b0), min(o + n, b1)
        if lo < hi:
            out.append((i, lo, hi))
    return out


def block_runs(offsets: Sequence[int], numels: Sequence[int], groups: Sequence[int], block: int,
               rank: int) -> List[Tuple[int, int, int, Optional[int]]]:
    """(lo, hi, group, index) tiling rank's block [0, block) in block coordinates: the part of parameter ``index`` (of
    parameter group ``group``) there, then the pad as (lo, block, B2_OPT_NO_GROUP, None), which is never stepped."""
    runs: List[Tuple[int, int, int, Optional[int]]] = [
        (lo - rank * block, hi - rank * block, groups[i], i) for i, lo, hi in block_intersections(offsets, numels, block, rank)]
    end = runs[-1][1] if runs else 0
    if end < block:
        runs.append((end, block, N.B2_OPT_NO_GROUP, None))
    return runs


def launch_runs(runs: Sequence[tuple], sgd: bool) -> List[Tuple[int, int, float, Optional[Tuple[int, bool]]]]:
    """(begin, group, step, pos) of one launch from (begin, group, steps taken or None for the pad[, pos]): the step a run's
    update uses (Adam: steps taken + 1; SGD: 1.0 on the first step, else 0.0; the pad: 0.0), adjacent equal runs
    coalesced.  ``pos`` = (index within its parameter of the run's first element, the parameter takes the fused Adam's
    scalar path) marks a run whose rounding depends on where its elements sit in their parameter (Adam's coupled weight
    decay, DESIGN.md 2.4): such a run is never merged."""
    out: List[Tuple[int, int, float, Optional[Tuple[int, bool]]]] = []
    for lo, gi, n, *rest in runs:
        pos = rest[0] if rest else None
        step = 0.0 if n is None else (float(n == 0) if sgd else float(n + 1))
        if pos is None and out and out[-1][1] == gi and out[-1][2] == step and out[-1][3] is None:
            continue
        out.append((lo, gi, step, pos))
    return out


def _check_run_bound(groups: Sequence[Sequence[int]], counts: Sequence[Sequence[int]], sgd: bool,
                     distinct: Optional[Sequence[Sequence[bool]]] = None) -> None:
    """Overlap mode: every launch's run table fits B2_OPT_MAX_RUNS.  A rank's block holds at most the runs of the whole
    bucket (adjacent parameters of one group and step coalesced) plus the pad, whatever W and the rank: checked from the
    bucket layout alone, so every rank reaches the same decision before any bucket is launched."""
    for bi, (gs, cs) in enumerate(zip(groups, counts)):
        ds = distinct[bi] if distinct is not None else [False] * len(gs)
        n = len(launch_runs([(0, g, c, (0, False) if d else None) for g, c, d in zip(gs, cs, ds)], sgd)) + 1
        if n > N.B2_OPT_MAX_RUNS:
            raise ValueError(
                f"overlap_with_ddp=True: bucket {bi} alternates between parameter groups (or step counts) {n - 1} times; the "
                f"fused step's run table holds {N.B2_OPT_MAX_RUNS - 1} runs and the pad.  Use a smaller bucket_cap_mb or "
                "order the parameters so that each group's are adjacent")


def _ordered(comm: Any, launch) -> None:
    from torchx_b200.nn.batchnorm import _ordered as ordered

    ordered(comm, launch)


class ZeroRedundancyOptimizer(torch.optim.Optimizer):
    """``optimizer_class`` (SGD, Adam or AdamW, with any of their options) over this rank's shard of a mini-DDP's
    parameters.  Constructing it switches ``model`` into sharded mode, which must happen before its first backward.

    ``params`` defaults to every trainable parameter of the model; torch-style groups over those parameters are accepted,
    and every trainable parameter must be in exactly one group.  ``param_groups`` are the inner optimizer's groups, so
    ``torch.optim.lr_scheduler`` works.

    After a synced backward the model parameters' ``.grad`` are None (the reduced gradients exist only as the shards), so
    clip with ``clip_grad_norm_`` of this class: ``torch.nn.utils.clip_grad_norm_(model.parameters(), ...)`` sees no
    gradients and clips nothing."""

    _step_supports_amp_scaling = True  # GradScaler hands itself to step(): the found-inf decision is made rank-global there

    def __init__(self, model: DistributedDataParallel, optimizer_class: type, params: Optional[Any] = None,
                 overlap_with_ddp: bool = False, **defaults: Any) -> None:
        if optimizer_class not in SUPPORTED:
            raise TypeError(f"ZeroRedundancyOptimizer supports {', '.join(c.__name__ for c in SUPPORTED)}, "
                            f"not {getattr(optimizer_class, '__name__', optimizer_class)}")
        if not isinstance(model, DistributedDataParallel):
            raise TypeError("ZeroRedundancyOptimizer shards a torchx_b200.ddp.DistributedDataParallel")
        if overlap_with_ddp and model.find_unused_parameters:
            raise ValueError(
                "overlap_with_ddp=True cannot be combined with find_unused_parameters=True: each bucket's step runs inside "
                "its reduce-scatter, before the ranks know which parameters none of them used, so such a parameter would be "
                "stepped with a zero gradient instead of skipped")
        groups = _normalize_groups(model._params if params is None else params)
        _check_groups(groups, model._params)
        if overlap_with_ddp:
            model._check_shardable()
            _check_overlap(groups, defaults, model)
            gi_of = {id(p): gi for gi, g in enumerate(groups) for p in g["params"]}
            pos = [optimizer_class is torch.optim.Adam and bool({**defaults, **g}.get("weight_decay", 0)) for g in groups]
            _check_run_bound([[gi_of[id(p)] for p in b.params] for b in model.buckets],
                             [[0] * len(b.params) for b in model.buckets], optimizer_class is torch.optim.SGD,
                             [[pos[gi_of[id(p)]] for p in b.params] for b in model.buckets])
        else:
            _check_split_params(optimizer_class, groups, defaults, model)
        super().__init__(groups, defaults)  # validates the groups and fills in the defaults
        self.model = model
        self.comm = model.comm
        self.optimizer_class = optimizer_class
        self.overlap_with_ddp = overlap_with_ddp
        self._full_groups = [list(g["params"]) for g in self.param_groups]  # model parameters, the user's order
        model._enable_sharding(self if overlap_with_ddp else None)

        W, r = model.world_size, self.comm.rank
        where: Dict[int, Tuple[Any, int, int]] = {}  # id(param) -> (bucket, offset, numel)
        for b in model.buckets:
            for p, o, n in zip(b.params, b.spec.offsets, b.spec.numels):
                where[id(p)] = (b, o, n)
        self._where = where
        # views[id(param)] = (view of the flat parameter buffer, bucket elements lo, hi): this rank's slice of it
        self._views: Dict[int, Tuple[torch.Tensor, int, int]] = {}
        for b in model.buckets:
            for i, lo, hi in block_intersections(b.spec.offsets, b.spec.numels, b.block, r):
                v = b.param_flat[lo:hi]
                self._views[id(b.params[i])] = (v, lo, hi)
                if not overlap_with_ddp:
                    model._shard_grads.append((v, b.shard_grad[lo - r * b.block : hi - r * b.block], b.params[i]))
        inner_groups = []
        for g, ps in zip(self.param_groups, self._full_groups):
            inner = {k: val for k, val in g.items() if k != "params"}
            inner["params"] = [self._views[id(p)][0] for p in ps if id(p) in self._views]
            inner_groups.append(inner)
        self.optim = optimizer_class(inner_groups, **defaults)
        self.param_groups = self.optim.param_groups  # scheduler writes reach the inner optimizer
        self.state = self.optim.state
        self.defaults = self.optim.defaults
        self._world, self._rank = W, r
        self._stepped = False  # the same on every rank: the skip decision under a GradScaler is rank-global
        self._stepped_in_backward = False  # overlap mode: a synced backward has updated this rank's blocks since step()
        if overlap_with_ddp:
            self._init_overlap()

    # ---- overlap_with_ddp: the step inside each bucket's reduce-scatter ---------------------------------------------
    def _init_overlap(self) -> None:
        """Flat per-bucket state buffers of ``block`` elements, which the kernel indexes like this rank's parameter block;
        the inner optimizer's per-parameter state entries are views into them, so checkpoints see the usual layout."""
        sgd = self.optimizer_class is torch.optim.SGD
        self._state_keys = ["momentum_buffer"] if sgd else ["exp_avg", "exp_avg_sq"]
        self._kind = N.B2_OPT_SGD if sgd else (N.B2_OPT_ADAM if self.optimizer_class is torch.optim.Adam else N.B2_OPT_ADAMW)
        group_of = {id(p): gi for gi, ps in enumerate(self._full_groups) for p in ps}
        dev, r = self.model.device, self._rank
        self._flat_state: Dict[int, Dict[str, torch.Tensor]] = {}
        self._runs: Dict[int, List[Tuple[int, int, int, Optional[torch.Tensor]]]] = {}
        self._count: Dict[int, int] = {}  # id(view) -> steps taken (host copy of the `step` state, no device sync)
        self._pos: Dict[int, Tuple[int, bool]] = {}  # id(view) -> (index in its parameter of its first element, scalar path)
        for bi, b in enumerate(self.model.buckets):
            flat = {k: torch.zeros(b.block, dtype=torch.float32, device=dev) for k in self._state_keys}
            self._flat_state[bi] = flat
            runs = []
            for lo, hi, gi, i in block_runs(b.spec.offsets, b.spec.numels, [group_of[id(p)] for p in b.params], b.block, r):
                v = self._views[id(b.params[i])][0] if i is not None else None
                runs.append((lo, hi, gi, v))
                if v is not None:  # where the run starts in its parameter, and whether the fused Adam's path is the scalar one
                    self._pos[id(v)] = (lo + r * b.block - b.spec.offsets[i], b.spec.numels[i] % 4 != 0)
                if v is not None:
                    self._count[id(v)] = 0
            self._runs[bi] = runs
        self._bucket_index = {id(b): bi for bi, b in enumerate(self.model.buckets)}
        self._attach_state()

    def _attach_state(self) -> None:
        """state[view] <- views of the flat buffers (and a device fp32 ``step``, as the fused optimizers keep it)."""
        for bi, runs in self._runs.items():
            for lo, hi, gi, v in runs:
                if v is None:
                    continue
                g = self.param_groups[gi]
                st: Dict[str, Any] = {}
                if self.optimizer_class is torch.optim.SGD:
                    if g["momentum"] != 0:
                        st["momentum_buffer"] = self._flat_state[bi]["momentum_buffer"][lo:hi]
                else:
                    st["step"] = torch.tensor(float(self._count[id(v)]), dtype=torch.float32, device=self.model.device)
                    st["exp_avg"] = self._flat_state[bi]["exp_avg"][lo:hi]
                    st["exp_avg_sq"] = self._flat_state[bi]["exp_avg_sq"][lo:hi]
                self.optim.state[v] = st

    def _launch_table(self, b) -> "N.B2Optim":
        """The b2_optim_t of one bucket launch: this rank's parameter and state blocks, its runs (adjacent parameters of
        one group and step count coalesced) and every group's hyper-parameters as param_groups hold them now."""
        bi = self._bucket_index[id(b)]
        t = N.B2Optim()
        t.kind = self._kind
        t.n_groups = len(self.param_groups)
        t.param = b.param_flat[self._rank * b.block :].data_ptr()
        flat = self._flat_state[bi]
        t.state0 = flat[self._state_keys[0]].data_ptr()
        t.state1 = flat["exp_avg_sq"].data_ptr() if "exp_avg_sq" in flat else None
        sgd = self._kind == N.B2_OPT_SGD
        for gi, g in enumerate(self.param_groups):
            h = t.group[gi]
            h.lr, h.weight_decay, h.maximize = float(g["lr"]), float(g["weight_decay"]), int(bool(g["maximize"]))
            if sgd:
                h.momentum, h.dampening, h.nesterov = float(g["momentum"]), float(g["dampening"]), int(bool(g["nesterov"]))
            else:
                h.beta1, h.beta2 = float(g["betas"][0]), float(g["betas"][1])
                h.eps = float(g["eps"])
        pos_groups = {gi for gi, g in enumerate(self.param_groups) if self._kind == N.B2_OPT_ADAM and g["weight_decay"]}
        runs = launch_runs([(lo, gi, self._count[id(v)] if v is not None else None,
                             self._pos[id(v)] if v is not None and gi in pos_groups else None)
                            for lo, _, gi, v in self._runs[bi]], sgd)
        assert len(runs) <= N.B2_OPT_MAX_RUNS, "bounded by _check_run_bound at construction and on load"
        t.n_runs = len(runs)
        for k, (lo, gi, step, pos) in enumerate(runs):
            t.run_begin[k], t.run_group[k], t.run_step[k] = lo, gi, step
            if pos is not None:
                t.run_index[k], t.run_scalar[k] = pos
        t.run_begin[len(runs)] = b.block
        return t

    # ---- step ------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None, grad_scaler=None):  # noqa: D401
        """Inner step on this rank's shard, then an in-place all-gather of every bucket's parameter buffer.  Under a
        GradScaler the found-inf flags are first reduced with MAX over the ranks, in the very tensors ``update()`` reads,
        so an inf in one rank's shard makes every rank skip the step and back off its scale alike.

        This relies on GradScaler passing itself as ``grad_scaler`` (torch 2.11 warns that the keyword is deprecated).  Its
        replacement hands the optimizer only a sum of the found-inf tensors, a new tensor, while ``update()`` reads the
        per-device ones: a MAX reduced into that sum would not reach the scale update, and the ranks' scales would drift
        apart.  Should torch drop the keyword, ``step()`` stops being called with it and a GradScaler run raises below."""
        if closure is not None:
            raise RuntimeError("ZeroRedundancyOptimizer.step does not take a closure")
        if self.overlap_with_ddp:
            return self._step_overlap(grad_scaler)
        if grad_scaler is None and getattr(self, "found_inf", None) is not None:
            raise RuntimeError("this GradScaler no longer passes itself to step(): the rank-global inf check cannot run")
        if grad_scaler is not None:
            from torch.amp.grad_scaler import OptState

            st = grad_scaler._per_optimizer_states[id(self)]
            if st["stage"] is OptState.READY:
                grad_scaler.unscale_(self)
            found = st["found_inf_per_device"]
            if not found:  # this rank holds no gradient: it still takes part in the reduction
                found[self.model.device] = torch.zeros((), dtype=torch.float32, device=self.model.device)
            for t in found.values():
                _ordered(self.comm, lambda s, t=t: self.comm.allreduce_op_(t, "max", stream=s))
            if sum(t.item() for t in found.values()):
                return None
        self.optim.step()
        self._stepped = True
        for b in self.model.buckets:
            own = b.param_flat[self._rank * b.block : (self._rank + 1) * b.block]
            _ordered(self.comm, lambda s, b=b, own=own: self.comm.allgather_(b.param_flat, own, stream=s))
        return None

    def _step_overlap(self, grad_scaler) -> None:
        """The update already ran inside the backward's reduce-scatters: all-gather every bucket's parameter buffer and
        advance the step counts.  A no-op without a synced backward since the previous step()."""
        if grad_scaler is not None or getattr(self, "found_inf", None) is not None:
            raise RuntimeError(
                "overlap_with_ddp=True does not support GradScaler: dynamic loss scaling needs the rank-global found-inf "
                "before any update, and with overlap the update has already happened during backward")
        if not self._stepped_in_backward:
            return None
        self._stepped_in_backward = False
        steps = []
        for k in self._count:
            self._count[k] += 1
        for st in self.optim.state.values():
            if "step" in st:
                steps.append(st["step"])
        if steps:
            torch._foreach_add_(steps, 1.0)
        self._stepped = True
        for b in self.model.buckets:
            own = b.param_flat[self._rank * b.block : (self._rank + 1) * b.block]
            _ordered(self.comm, lambda s, b=b, own=own: self.comm.allgather_(b.param_flat, own, stream=s))
        return None

    def zero_grad(self, set_to_none: bool = True) -> None:
        """Clears the gradient shards and the model parameters' ``.grad``.  Required between a step and the next synced
        backward: the reduced gradients live only in the shards, which a synced backward overwrites (it raises instead)."""
        self.model._shard_grads_live = False
        for v, g, _ in self.model._shard_grads:
            if set_to_none:
                v.grad = None
            else:
                g.zero_()
                v.grad = g
        for p in self.model._params:
            if set_to_none:
                p.grad = None
            elif p.grad is not None:
                p.grad.detach_().zero_()

    @torch.no_grad()
    def clip_grad_norm_(self, max_norm: float) -> torch.Tensor:
        """Clips the sharded gradients in place by their global 2-norm and returns that norm (fp32, the same bits on
        every rank): the sqrt of the rank-order fp32 sum of each rank's fp32 sum of squares over its shard.  The clip
        coefficient is torch's, ``max_norm / (norm + 1e-6)`` clamped to 1."""
        if self.overlap_with_ddp:
            raise RuntimeError("overlap_with_ddp=True does not support clip_grad_norm_: the update has already happened "
                               "during backward, before a global norm could be known")
        dev = self.model.device
        grads = [v.grad for v, _, _ in self.model._shard_grads if v.grad is not None]
        sq = torch.zeros(1, dtype=torch.float32, device=dev)
        if grads:
            sq = torch.stack([g.float().square().sum() for g in grads]).sum().reshape(1)
        _ordered(self.comm, lambda s: self.comm.allreduce_op_(sq, "sum", stream=s))
        norm = sq.sqrt()[0]
        coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
        if grads:
            torch._foreach_mul_(grads, coef.to(grads[0].dtype))
        return norm

    # ---- checkpoints -----------------------------------------------------------------------------
    def _index(self) -> List[torch.nn.Parameter]:
        return [p for ps in self._full_groups for p in ps]  # the unsharded optimizer's param index order

    def _keys(self, group: Dict[str, Any]) -> List[str]:
        """Per-parameter state keys of a group once it has stepped, in the order the optimizer class creates them."""
        if self.optimizer_class is torch.optim.SGD:
            return ["momentum_buffer"] if group["momentum"] != 0 else []
        return ["step", "exp_avg", "exp_avg_sq"] + (["max_exp_avg_sq"] if group["amsgrad"] else [])

    def consolidate_state_dict(self, to: int = 0) -> None:
        """Collective: all-gathers every rank's state slices (exact bytes) so that ``state_dict()`` on rank ``to``
        returns the state dict the unsharded optimizer would have, in host memory (as torch's ZeroRedundancyOptimizer
        keeps it).  On the GPU only one bucket of one state at a time is ever full-size; the other ranks keep nothing."""
        self._consolidated = None  # an earlier checkpoint's copy is not held alongside this one
        params = self._index()
        r, W, dev = self._rank, self._world, self.model.device
        keys_of = {id(p): self._keys(g) if self._stepped else [] for g, ps in zip(self.param_groups, self._full_groups) for p in ps}
        tensor_keys = [k for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "momentum_buffer")
                       if any(k in ks for ks in keys_of.values())]
        # Adam's scalar `step`: one fp32 per parameter from every rank, taken from the lowest rank that holds a slice, and
        # after them a 1 for each parameter whose slice here has state (one that never had a gradient, unused on every rank
        # since the start, has none, as in the unsharded optimizer).  Read before any collective is issued, so that no host
        # sync waits behind them.
        n = len(params)
        own_steps = torch.zeros(2 * n, dtype=torch.float32, device=dev)
        for i, p in enumerate(params):
            st = self.optim.state.get(self._views[id(p)][0], {}) if id(p) in self._views else {}
            if st.get("step") is not None:
                own_steps[i : i + 1].copy_(st["step"].reshape(1), non_blocking=True)
            if st:
                own_steps[n + i] = 1.0
        n2 = 2 * n
        steps = torch.zeros(W * n2, dtype=torch.float32, device=dev)
        steps[r * n2 : (r + 1) * n2].copy_(own_steps)
        full: Dict[str, Dict[int, torch.Tensor]] = {k: {} for k in tensor_keys}
        for k in tensor_keys:
            for b in self.model.buckets:
                buf = torch.zeros(W * b.block, dtype=b.dtype, device=dev)
                for p in b.params:
                    if id(p) in self._views:
                        v, lo, hi = self._views[id(p)]
                        st = self.optim.state.get(v, {}).get(k)
                        if st is not None:
                            buf[lo:hi].copy_(st)
                own = buf[r * b.block : (r + 1) * b.block]
                _ordered(self.comm, lambda s, buf=buf, own=own: self.comm.allgather_(buf, own, stream=s))
                if r == to:
                    host = buf.cpu()
                    for p, o, numel in zip(b.params, b.spec.offsets, b.spec.numels):
                        full[k][id(p)] = _view_like(host[o : o + numel], p).clone()
                del buf, own
        _ordered(self.comm, lambda s: self.comm.allgather_(steps, steps[r * n2 : (r + 1) * n2], stream=s))
        if r != to:
            return
        steps_h = steps.view(W, n2).cpu()
        has_state = steps_h[:, n:].amax(0) > 0
        state: Dict[int, Dict[str, Any]] = {}
        for i, p in enumerate(params):
            entry: Dict[str, Any] = {}
            for k in keys_of[id(p)] if has_state[i] else []:
                if k == "step":
                    owner = next(q for q in range(W) if _owns(self._where[id(p)], q))
                    entry[k] = steps_h[owner, i].clone()
                else:
                    entry[k] = full[k][id(p)]
            if entry:
                state[i] = entry
        groups, at = [], 0
        for g, ps in zip(self.param_groups, self._full_groups):
            d = {k: val for k, val in g.items() if k != "params"}
            d["params"] = list(range(at, at + len(ps)))
            at += len(ps)
            groups.append(d)
        self._consolidated = {"state": state, "param_groups": groups}

    def state_dict(self) -> Dict[str, Any]:
        """After ``consolidate_state_dict(to)``, on rank ``to``: the state dict of the unsharded optimizer (its
        param_groups and param indices; full-size per-parameter state)."""
        sd = getattr(self, "_consolidated", None)
        if sd is None:
            raise RuntimeError("call consolidate_state_dict(to) on every rank first; state_dict() returns on rank `to` only")
        return sd

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        """Loads the full (unsharded) form on every rank, keeping this rank's slices."""
        groups = state_dict["param_groups"]
        if len(groups) != len(self._full_groups) or any(len(g["params"]) != len(ps) for g, ps in zip(groups, self._full_groups)):
            raise ValueError("the state dict's param groups do not match this optimizer's")
        if self.overlap_with_ddp:
            self._check_loaded_runs(state_dict)
        inner_state: Dict[int, Dict[str, Any]] = {}
        inner_groups, at = [], 0
        for g, ps in zip(groups, self._full_groups):
            d = {k: val for k, val in g.items() if k != "params"}
            d["params"] = []
            for idx, p in zip(g["params"], ps):
                if id(p) not in self._views:
                    continue
                v, lo, hi = self._views[id(p)]
                o = self._where[id(p)][1]
                entry = {}
                for k, val in state_dict["state"].get(idx, {}).items():
                    if k != "step" and torch.is_tensor(val):  # per-element state (a 0-dim parameter's too): this rank's slice
                        mem = _view_like(torch.empty(p.numel(), dtype=val.dtype, device=p.device), p)
                        mem.copy_(val)  # the parameter's memory order, as the flat buffer holds it
                        val = mem.as_strided((p.numel(),), (1,))[lo - o : hi - o]
                    entry[k] = val.clone() if torch.is_tensor(val) else val  # never alias the caller's state
                if entry:
                    inner_state[at] = entry
                d["params"].append(at)
                at += 1
            inner_groups.append(d)
        self.optim.load_state_dict({"state": inner_state, "param_groups": inner_groups})
        self._stepped = bool(state_dict["state"])
        self.param_groups = self.optim.param_groups
        self.state = self.optim.state
        if self.overlap_with_ddp:
            self._land_loaded_state()

    def _check_loaded_runs(self, state_dict: Dict[str, Any]) -> None:
        """Overlap mode, before loading: the run bound with the checkpoint's step counts (the same on every rank)."""
        index = {id(p): i for i, p in enumerate(self._index())}
        gi_of = {id(p): gi for gi, ps in enumerate(self._full_groups) for p in ps}
        sgd = self.optimizer_class is torch.optim.SGD

        def count(p):
            st = state_dict["state"].get(index[id(p)], {})
            return int(float(st["step"])) if "step" in st else int(bool(st))

        pos = [self._kind == N.B2_OPT_ADAM and bool(g["weight_decay"]) for g in self.param_groups]
        _check_run_bound([[gi_of[id(p)] for p in b.params] for b in self.model.buckets],
                         [[count(p) for p in b.params] for b in self.model.buckets], sgd,
                         [[pos[gi_of[id(p)]] for p in b.params] for b in self.model.buckets])

    @torch.no_grad()
    def _land_loaded_state(self) -> None:
        """Overlap mode: the loaded per-parameter state goes into the flat buffers the kernel steps, and the state entries
        become views of them again; the host step counts follow the loaded ``step`` (read once, here)."""
        loaded = {id(v): st for v, st in self.optim.state.items()}
        for flat in self._flat_state.values():
            for t in flat.values():
                t.zero_()
        for bi, runs in self._runs.items():
            for lo, hi, gi, v in runs:
                if v is None:
                    continue
                st = loaded.get(id(v), {})
                for k in self._state_keys:
                    if k in st:
                        self._flat_state[bi][k][lo:hi].copy_(st[k].reshape(-1))
                if "step" in st:
                    self._count[id(v)] = int(float(st["step"]))
                else:
                    self._count[id(v)] = 1 if st else 0
        self.optim.state.clear()
        self._attach_state()


def _check_overlap(groups: List[Dict[str, Any]], defaults: Dict[str, Any], model: DistributedDataParallel) -> None:
    """What the fused step inside the reduce-scatter cannot do, refused before anything is sharded."""
    if model.wire not in ("bf16", "f32", "f16"):
        raise ValueError(f"overlap_with_ddp=True: unknown wire format {model.wire!r}")
    if any(p.dtype != torch.float32 for p in model._params):
        raise TypeError("overlap_with_ddp=True steps fp32 parameters only (modes B2_F32_WIRE_BF16, B2_F32, B2_F32_WIRE_F16)")
    if len(groups) > N.B2_OPT_MAX_GROUPS:
        raise ValueError(f"overlap_with_ddp=True takes at most {N.B2_OPT_MAX_GROUPS} parameter groups, got {len(groups)}")
    for g in groups:
        opts = {**defaults, **{k: v for k, v in g.items() if k != "params"}}
        if opts.get("amsgrad"):
            raise ValueError("overlap_with_ddp=True does not support amsgrad")
        if torch.is_tensor(opts.get("lr")):
            raise TypeError("overlap_with_ddp=True needs a float lr, not a tensor")
        if opts.get("foreach"):
            raise ValueError("overlap_with_ddp=True runs its own fused step: foreach=True does not apply")
        for k in ("capturable", "differentiable"):
            if opts.get(k):
                raise ValueError(f"overlap_with_ddp=True does not support {k}=True")


def _check_split_params(optimizer_class: type, groups: List[Dict[str, Any]], defaults: Dict[str, Any],
                        model: DistributedDataParallel) -> None:
    """Without overlap the inner optimizer steps one 1-D view per (parameter, rank block).  Two of torch's fused kernels do
    not step such views to the bits of the whole tensor when a block boundary splits a parameter of a numel that is not a
    multiple of 4 (the whole tensor takes their scalar path, a view of a multiple of 4 elements the vectorised one, and a
    view counts its elements from 0; DESIGN.md 2.4): Adam with coupled weight decay and without maximize, whose rounding of
    ``param * weight_decay`` depends on an element's index, and SGD with maximize, momentum and no weight decay, whose
    momentum update is contracted differently on the two paths.  Refused here, from the bucket layout alone, so every rank
    raises alike before anything is sharded."""
    W = model.world_size
    names = {id(p): n for n, p in model.module.named_parameters()}
    gi_of = {id(p): gi for gi, g in enumerate(groups) for p in g["params"]}
    what = []
    for g in groups:
        o = {**defaults, **g}
        if not o.get("fused"):
            what.append(None)
        elif optimizer_class is torch.optim.Adam and o.get("weight_decay", 0) and not o.get("maximize"):
            what.append("Adam(fused=True) with weight_decay")
        elif (optimizer_class is torch.optim.SGD and o.get("maximize") and o.get("momentum", 0)
              and not o.get("weight_decay", 0)):
            what.append("SGD(fused=True) with maximize, momentum and no weight_decay")
        else:
            what.append(None)
    for b in model.buckets:
        B = padded_block(b.spec.numel, W)
        for p, off, n in zip(b.params, b.spec.offsets, b.spec.numels):
            w = what[gi_of[id(p)]]
            if w is None or n % 4 == 0 or off // B == (off + n - 1) // B:
                continue
            fix = ("overlap_with_ddp=True (whose fused step is exact here) or foreach=True" if optimizer_class is torch.optim.Adam
                   else "foreach=True")
            raise ValueError(
                f"ZeroRedundancyOptimizer: parameter {names.get(id(p), '?')!r} ({n} elements, not a multiple of 4) is split "
                f"between rank blocks, and {w} would step its pieces to other bits than the whole tensor; use {fix}")


def _owns(where, rank: int) -> bool:
    b, o, n = where
    return max(o, rank * b.block) < min(o + n, (rank + 1) * b.block)


def _normalize_groups(params: Any) -> List[Dict[str, Any]]:
    params = list(params)
    if not params:
        raise ValueError("ZeroRedundancyOptimizer got an empty parameter list")
    if not isinstance(params[0], dict):
        params = [{"params": params}]
    return [dict(g, params=list(g["params"])) for g in params]


def _check_groups(groups: List[Dict[str, Any]], trainable: Sequence[torch.nn.Parameter]) -> None:
    """Every trainable parameter of the model in exactly one group, and nothing else."""
    want = {id(p) for p in trainable}
    seen = set()
    for g in groups:
        for p in g["params"]:
            if id(p) not in want:
                raise ValueError("a parameter group holds a tensor that is not a trainable parameter of the model")
            if id(p) in seen:
                raise ValueError("a parameter appears in more than one group (or twice in one)")
            seen.add(id(p))
    if seen != want:
        raise ValueError(f"{len(want - seen)} trainable parameters of the model are in no parameter group")
