"""find_unused_parameters=True in the mini-DDP and its ZeRO-1 mode, on the GPU.

Two processes on cuda:0 (gloo for stock DDP's bookkeeping): the mini-DDP against stock DistributedDataParallel with
find_unused_parameters=True, gradients and parameters bit for bit and the same parameters left without a gradient
(tests/workers/unused_worker.py).  In-process at W = 2 and 4: a model that uses every parameter gives the bits and bucket
kernels of find_unused_parameters=False, and the oracle's; sharded ZeRO-1 under an unused pattern is bit-equal to the
unsharded mini-DDP over several steps and a checkpoint round trip.

The in-process ranks run ONE backward over all their losses: each rank's _finalize_backward may wait on the host for the
used map's reduction, which needs every rank's launch, and the final callbacks of one backward run after all its hooks."""
import os
import socket
import subprocess
import sys
import uuid

import pytest
import torch
from torch import nn

import oracle
from tests._util import assert_bits_equal
from tests.test_zero_gpu import _assert_same, _assert_state_equal, _consolidate, _ddps, _params, _phase

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_matches_stock_ddp_two_ranks_one_gpu(tmp_path):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    shm = f"/b2_unused_{uuid.uuid4().hex[:12]}"
    procs = []
    for r in range(2):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "unused_worker.py"), "--rank", str(r), "--world", "2",
               "--shm", shm, "--port", str(port)]
        procs.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            o, _ = p.communicate(timeout=600)
            outs.append(o)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, p in enumerate(procs):
        assert p.returncode == 0, f"rank {r} failed:\n{outs[r]}"
    print(outs[0])


class _Heads(nn.Module):
    """A trunk and three heads; forward(x, use) runs the heads whose bit is set in `use`.  Sizes are multiples of 16 (the
    flat buffer keeps each parameter 64-byte aligned, see tests/test_zero_gpu.py) except one 13-element bias, which a
    rank block boundary splits at W = 2 and 4."""

    def __init__(self):
        super().__init__()
        self.trunk = nn.Linear(32, 64)
        self.heads = nn.ModuleList([nn.Linear(64, 16), nn.Linear(64, 13), nn.Linear(64, 16)])

    def forward(self, x, use=0b111):
        h = self.trunk(x).relu()
        outs = [head(h) for k, head in enumerate(self.heads) if use >> k & 1]
        return {"out": outs, "h": h}


def _model(seed):
    torch.manual_seed(seed)
    return _Heads().cuda()


def _loss(out):
    return sum(o.square().mean() for o in out["out"]) + 0.01 * out["h"].mean()


def _x(r, step):
    return torch.randn(16, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1000 * step + r))


def _backward_all(ddps, streams, step, use, opts=None):
    """Every rank's forward on its stream, then one backward over all the losses (see the module docstring)."""
    losses = []
    for r, (d, s) in enumerate(zip(ddps, streams)):
        with torch.cuda.stream(s):
            if opts is not None:
                opts[r].zero_grad()
            losses.append(_loss(d(_x(r, step), use(r, step))))
    torch.autograd.backward(losses)
    torch.cuda.synchronize()


def _warm(ddps, streams):
    """Loads every kernel the ranks' backwards and the used map's MAX reduction run before any rank waits on another.  On
    a twin of the model: a no_sync backward of the DDP would count as a use of every parameter in the next synced one."""
    t = _model(0)
    _loss(t(_x(0, 99))).backward()
    grads = [p.grad for p in t.parameters()]
    torch._foreach_copy_(grads, grads)
    torch._foreach_zero_(grads)
    torch.cuda.synchronize()
    _phase(len(ddps), lambda r: ddps[r].comm.allreduce_op_(torch.zeros(5, dtype=torch.int32, device="cuda"), "max",
                                                            stream=streams[r]))


def _on(stream, fn):
    with torch.cuda.stream(stream):
        fn()


def _flat_grads(module):
    return torch.cat([p.grad.reshape(-1) for p in module.parameters()]).cpu().numpy()


@pytest.mark.parametrize("W", [2, 4])
def test_every_parameter_used_gives_the_bits_and_kernels_of_the_default(W):
    ca, off, sa = _ddps(W, _model)
    cb, on, sb = _ddps(W, _model, find_unused_parameters=True)
    try:
        twins = [_model(0) for _ in range(W)]
        _warm(off, sa)
        _warm(on, sb)
        launches = [c.launches for c in ca + cb]
        for step in range(3):
            _backward_all(off, sa, step, lambda r, s: 0b111)
            _backward_all(on, sb, step, lambda r, s: 0b111)
            local = []
            for r, t in enumerate(twins):
                t.zero_grad(set_to_none=True)
                _loss(t(_x(r, step))).backward()
                local.append(_flat_grads(t))
            want = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, local, 1.0 / W)
            for r in range(W):
                assert_bits_equal(_flat_grads(on[r].module), want, f"find_unused_parameters=True step {step} rank {r}")
                assert_bits_equal(_flat_grads(off[r].module), want, f"find_unused_parameters=False step {step} rank {r}")
            for d in off + on:
                d.zero_grad(set_to_none=True)
        for a, b in zip(off, on):
            assert (a.gathered_buckets, a.copied_in_buckets) == (b.gathered_buckets, b.copied_in_buckets)
        n = len(ca)
        grew = [c.launches - l0 for c, l0 in zip(ca + cb, launches)]
        assert grew[n:] == [g + 3 for g in grew[:n]], grew  # the same bucket kernels, plus one used-map MAX per backward
    finally:
        for c in ca + cb:
            c.close()


def _use(r, step):
    """Head 0 always; head 1 on rank 0 at even steps and on rank 1 at step 1 (locally unused, globally used), on no rank
    at step 3 (globally unused); head 2 never."""
    return 0b001 | (0b010 if (r == 0 and step % 2 == 0) or (r == 1 and step == 1) else 0)


OPTS = {"sgd": (torch.optim.SGD, dict(lr=0.05, momentum=0.9, weight_decay=0.01)),
        "adamw": (torch.optim.AdamW, dict(lr=1e-2, weight_decay=0.05))}


@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("zero_copy", [True, False])
def test_sharded_is_bit_equal_to_unsharded_with_unused_parameters(W, opt, zero_copy):
    from torchx_b200.ddp import ZeroRedundancyOptimizer
    from torchx_b200.ddp.zero import padded_block

    cls, kw = OPTS[opt]
    ca, plain_ddps, sa = _ddps(W, _model, find_unused_parameters=True, zero_copy=zero_copy)
    cb, zero_ddps, sb = _ddps(W, _model, find_unused_parameters=True, zero_copy=zero_copy)
    try:
        split = False  # a block boundary inside a parameter
        for b in plain_ddps[0].buckets:
            B = padded_block(b.spec.numel, W)
            split |= any(o // B != (o + n - 1) // B for o, n in zip(b.spec.offsets, b.spec.numels))
        assert split
        plain = [cls(d.parameters(), **kw) for d in plain_ddps]
        zero = [ZeroRedundancyOptimizer(d, cls, **kw) for d in zero_ddps]
        _warm(plain_ddps, sa)
        _warm(zero_ddps, sb)
        dead = plain_ddps[0].module.heads[2]
        dead0 = [p.detach().clone() for p in dead.parameters()]
        for step in range(5):
            if step == 3:  # a checkpoint round trip between steps
                _consolidate(zero, 0, sb)
                sd = zero[0].state_dict()
                _assert_state_equal(sd, plain[0].state_dict(), f"state before step {step}")
                for z in zero:
                    z.load_state_dict(sd)
            _backward_all(plain_ddps, sa, step, _use, plain)
            _backward_all(zero_ddps, sb, step, _use, zero)
            for r in range(W):
                heads = plain_ddps[r].module.heads
                assert all(p.grad is None for p in heads[2].parameters()), "globally unused: no gradient"
                assert all((p.grad is None) == (step == 3) for p in heads[1].parameters()), step
                got = {id(v) for v, _, p in zero_ddps[r]._shard_grads if v.grad is not None}
                want = {id(v) for v, _, p in zero_ddps[r]._shard_grads
                        if not any(p is q for q in zero_ddps[r].module.heads[2].parameters())
                        and not (step == 3 and any(p is q for q in zero_ddps[r].module.heads[1].parameters()))}
                assert got == want, f"step {step} rank {r}: the shard views of globally unused parameters get no .grad"
            _phase(W, lambda r: _on(sa[r], plain[r].step))
            _phase(W, lambda r: _on(sb[r], zero[r].step))  # each rank on its own stream: the step's all-gathers wait for peers
            for r in range(W):
                _assert_same(_params(zero_ddps[r]), _params(plain_ddps[r]), f"{opt} W={W} step {step} rank {r}")
        _assert_same([p.detach() for p in dead.parameters()], dead0, "the globally unused head moved")
        _consolidate(zero, 0, sb)
        _assert_state_equal(zero[0].state_dict(), plain[0].state_dict(), "consolidated state")
    finally:
        for c in ca + cb:
            c.close()


def test_reachable_parameter_without_gradient_still_raises():
    """A parameter the output reaches but whose gradient never arrives (the backward stops short of it) is not unused."""
    ca, ddps, sa = _ddps(1, _model, find_unused_parameters=True)
    try:
        out = ddps[0](_x(0, 0))
        with pytest.raises(RuntimeError, match="never became ready"):
            torch.autograd.backward([o.square().mean() for o in out["out"]], inputs=list(ddps[0].module.heads.parameters()))
        torch.cuda.synchronize()
    finally:
        for c in ca:
            c.close()
