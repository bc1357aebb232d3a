"""torchx_b200.ddp.DistributedDataParallel and the comm hook against the oracle, all ranks in one process."""
import numpy as np
import pytest
import torch
from torch import nn

import oracle
from tests._util import assert_bits_equal

pytestmark = pytest.mark.gpu


def _mlp(seed):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(64, 256), nn.ReLU(), nn.Linear(256, 256), nn.ReLU(), nn.Linear(256, 16)).cuda()


def _flat_grads(m):
    return torch.cat([p.grad.reshape(-1) for p in m.parameters()]).cpu().numpy()


def _make_world(W, seeds, **kw):
    from torchx_b200.ddp import Communicator, DistributedDataParallel

    comms = Communicator.create_local([0] * W, stage_mb=8)
    for c in comms:
        c.set_timeout(20.0)
        c.set_max_ctas(4)
    # construction broadcasts rank 0's parameters: every rank's constructor must be in flight together, so build
    # them on side streams (the constructor enqueues its broadcast on the current stream)
    streams = [torch.cuda.Stream() for _ in range(W)]
    ddps = []
    for r in range(W):
        with torch.cuda.stream(streams[r]):
            ddps.append(DistributedDataParallel(_mlp(seeds[r]), comms[r], **kw))
    torch.cuda.synchronize()
    return comms, ddps, streams


@pytest.mark.parametrize("W", [2, 4])
def test_ddp_gradients_match_oracle_and_params_stay_in_sync(W):
    comms, ddps, streams = _make_world(W, seeds=list(range(W)), bucket_cap_mb=0.25, first_bucket_mb=0.05)
    try:
        assert len(ddps[0].buckets) >= 2
        ref0 = [p.detach().clone() for p in ddps[0].module.parameters()]
        for d in ddps[1:]:  # rank-0 broadcast at construction (distributed.py:881-890)
            for a, b in zip(ref0, d.module.parameters()):
                assert torch.equal(a, b)
        opts = [torch.optim.SGD(d.parameters(), lr=0.05, momentum=0.9) for d in ddps]
        for step in range(3):
            xs = [torch.randn(32, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(100 * step + r)) for r in range(W)]
            # local (un-synced) gradients of an identical replica
            local = []
            for r in range(W):
                twin = _mlp(0)
                twin.load_state_dict(ddps[r].module.state_dict())
                twin(xs[r]).square().mean().backward()
                local.append(_flat_grads(twin))
            for r in range(W):
                with torch.cuda.stream(streams[r]):
                    opts[r].zero_grad(set_to_none=True)
                    ddps[r](xs[r]).square().mean().backward()
            torch.cuda.synchronize()
            for c in comms:
                c.check()
            want = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, local, 1.0 / W)
            for r in range(W):
                assert_bits_equal(_flat_grads(ddps[r].module), want, f"step {step} rank {r}")
            for r in range(W):
                with torch.cuda.stream(streams[r]):
                    opts[r].step()
            torch.cuda.synchronize()
            p0 = [p.detach() for p in ddps[0].module.parameters()]
            for d in ddps[1:]:
                for a, b in zip(p0, d.module.parameters()):
                    assert torch.equal(a, b)
    finally:
        for c in comms:
            c.close()


def test_no_sync_accumulates_locally_and_fp32_wire():
    comms, ddps, streams = _make_world(2, seeds=[0, 0], wire="f32")
    try:
        xs = [torch.randn(8, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(r)) for r in range(2)]
        local = []
        for r in range(2):
            twin = _mlp(0)
            twin(xs[r]).sum().backward()
            twin(xs[r]).sum().backward()
            local.append(_flat_grads(twin))
        for r in range(2):
            with torch.cuda.stream(streams[r]):
                with ddps[r].no_sync():
                    ddps[r](xs[r]).sum().backward()
                ddps[r](xs[r]).sum().backward()
        torch.cuda.synchronize()
        want = oracle.allreduce(oracle.B2O_F32, local, 0.5)
        for r in range(2):
            assert_bits_equal(_flat_grads(ddps[r].module), want, f"rank {r}")
    finally:
        for c in comms:
            c.close()


def _run_ranks(W, fn):
    """One host thread per rank, like the real one-process-per-GPU topology: a host-side sync inside one rank's
    step (cuDNN handle/workspace setup, allocator) must not stop the other ranks from launching their kernels."""
    import threading

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


def test_buffers_follow_rank0_every_forward():
    from torchx_b200.ddp import Communicator, DistributedDataParallel

    comms = Communicator.create_local([0, 0], stage_mb=8)
    try:
        streams = [torch.cuda.Stream() for _ in range(2)]
        nets = []
        for r in range(2):
            comms[r].set_timeout(20.0)
            comms[r].set_max_ctas(8)
            torch.manual_seed(r)
            net = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.ReLU(), nn.Flatten(), nn.LazyLinear(4)).cuda()
            net(torch.zeros(2, 3, 8, 8, device="cuda"))  # materialise the lazy layer
            nets.append(net)
        torch.cuda.synchronize()
        ddps = [None, None]

        def build(r):
            with torch.cuda.stream(streams[r]):
                ddps[r] = DistributedDataParallel(nets[r], comms[r])
                streams[r].synchronize()

        _run_ranks(2, build)

        def train(r):
            with torch.cuda.stream(streams[r]):
                for step in range(2):
                    x = torch.randn(4, 3, 8, 8, device="cuda") * (r + 1)
                    ddps[r](x).sum().backward()
                ddps[r]._sync_buffers()  # what the next forward would do (distributed.py:2176-2243)
                streams[r].synchronize()

        _run_ranks(2, train)
        for c in comms:
            c.check()
        b0 = dict(ddps[0].module.named_buffers())
        assert b0["1.num_batches_tracked"].item() == 3  # lazy-init forward + 2 training forwards, rank 0's count
        for name, b in ddps[1].module.named_buffers():
            assert torch.equal(b, b0[name]), name
    finally:
        for c in comms:
            c.close()


def test_comm_hook_on_stock_ddp_world1():
    """hook(state, bucket) -> Future[Tensor] honoured on torch's own DistributedDataParallel (world 1: the fused
    kernel degenerates to the cast/scale pass, i.e. grads become float(bf16(g)))."""
    import os

    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as TorchDDP

    from torchx_b200.ddp import B200HookState, Communicator, b200_bf16_compress_hook

    import socket

    with socket.socket() as sock:  # any free port: a fixed one could collide with another job on the box
        sock.bind(("127.0.0.1", 0))
        port = sock.getsockname()[1]
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=0, world_size=1)
    comm = Communicator.create(0, 1, 0, "/unused")
    try:
        m = _mlp(0)
        twin = _mlp(0)
        d = TorchDDP(m, device_ids=[0])
        d.register_comm_hook(B200HookState(comm), b200_bf16_compress_hook)
        x = torch.randn(16, 64, device="cuda")
        d(x).square().mean().backward()
        twin(x).square().mean().backward()
        torch.cuda.synchronize()
        comm.check()
        want = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, [_flat_grads(twin)], 1.0)
        assert_bits_equal(_flat_grads(m), want, "hook")
    finally:
        comm.close()
        dist.destroy_process_group()


def _ragged_mlp(seed):
    torch.manual_seed(seed)
    # 37- and 13-wide layers: parameter sizes that are not multiples of 8, so later parameters start at bucket offsets that
    # are not vec-aligned (segment-straddling vecs in the zero-copy bucket fill).  No cuDNN here on purpose: an in-process
    # world cannot survive a first-use cudaMalloc / device-wide sync while a peer's kernel spins (the convnet / channels_last
    # variant runs one process per rank in tests/test_hook_multirank_gpu.py).
    return nn.Sequential(nn.Linear(64, 256), nn.ReLU(), nn.Linear(256, 37), nn.ReLU(), nn.Linear(37, 13)).cuda()


@pytest.mark.parametrize("zero_copy", [True, False])
def test_zero_copy_bucket_fill_equals_copy_in(zero_copy):
    """The kernel gathers the gradients straight from the per-parameter tensors (segment table in the kernel parameters) -
    same bits as copying them into the bucket first; ragged sizes, segment-straddling vecs, gradients that already ARE the
    bucket views (zero_grad(set_to_none=False))."""
    from torchx_b200.ddp import Communicator, DistributedDataParallel

    W = 2
    comms = Communicator.create_local([0] * W, stage_mb=8)
    try:
        streams = [torch.cuda.Stream() for _ in range(W)]
        ddps = []
        for r in range(W):
            comms[r].set_timeout(20.0)
            comms[r].set_max_ctas(4)
            with torch.cuda.stream(streams[r]):
                ddps.append(DistributedDataParallel(_ragged_mlp(0), comms[r], bucket_cap_mb=0.02, first_bucket_mb=0.002, zero_copy=zero_copy))
        torch.cuda.synchronize()
        assert len(ddps[0].buckets) >= 2
        for step in range(3):
            xs = [torch.randn(8, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(7 * step + r)) for r in range(W)]
            local = []
            for r in range(W):
                twin = _ragged_mlp(0)
                twin(xs[r]).square().mean().backward()
                local.append(_flat_grads(twin))
            for r in range(W):
                with torch.cuda.stream(streams[r]):
                    ddps[r].zero_grad(set_to_none=(step != 1))  # step 1: grads stay bucket views and accumulate in place
                    ddps[r](xs[r]).square().mean().backward()
            torch.cuda.synchronize()
            for c in comms:
                c.check()
            want = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, local, 1.0 / W)
            for r in range(W):
                assert_bits_equal(_flat_grads(ddps[r].module), want, f"step {step} rank {r}")
        if zero_copy:
            assert ddps[0].gathered_buckets > 0 and ddps[0].copied_in_buckets == 0
        else:
            assert ddps[0].gathered_buckets == 0
    finally:
        for c in comms:
            c.close()


def _grad_bits(m):
    """Flat gradients as bit patterns: bf16 as uint16, fp32 as float32."""
    g = torch.cat([p.grad.reshape(-1) for p in m.parameters()])
    return g.view(torch.int16).cpu().numpy().view(np.uint16) if g.dtype == torch.bfloat16 else g.cpu().numpy()


def _check_ddp_against_twins(W, make, mode, steps=2, **kw):
    """W ranks of DistributedDataParallel(make()) against the oracle on the gradients of un-synced twins; returns rank 0's
    DistributedDataParallel (for its bucket counters).  One warm-up backward per rank under no_sync() first, so that no
    first-use allocation happens on a rank's stream while a peer's kernel spins."""
    from torchx_b200.ddp import Communicator, DistributedDataParallel

    comms = Communicator.create_local([0] * W, stage_mb=8)
    try:
        streams = [torch.cuda.Stream() for _ in range(W)]
        ddps = []
        for r in range(W):
            comms[r].set_timeout(20.0)
            comms[r].set_max_ctas(4)
            with torch.cuda.stream(streams[r]):
                ddps.append(DistributedDataParallel(make(), comms[r], **kw))
        torch.cuda.synchronize()
        dtype = next(ddps[0].parameters()).dtype
        for r in range(W):
            with torch.cuda.stream(streams[r]), ddps[r].no_sync():
                ddps[r](torch.zeros(8, 64, device="cuda", dtype=dtype)).square().mean().backward()
                ddps[r].zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        for step in range(steps):
            xs = [torch.randn(8, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(11 * step + r)).to(dtype) for r in range(W)]
            local = []
            for r in range(W):
                twin = make()
                twin.load_state_dict(ddps[r].module.state_dict())
                twin(xs[r]).square().mean().backward()
                local.append(_grad_bits(twin))
            for r in range(W):
                with torch.cuda.stream(streams[r]):
                    ddps[r].zero_grad(set_to_none=True)
                    ddps[r](xs[r]).square().mean().backward()
            torch.cuda.synchronize()
            for c in comms:
                c.check()
            want = oracle.allreduce(mode, local, 1.0 / W)
            for r in range(W):
                assert_bits_equal(_grad_bits(ddps[r].module), want, f"step {step} rank {r}")
        return ddps[0]
    finally:
        for c in comms:
            c.close()


@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("algo", ["oneshot", "twoshot", "twoshot_pipe", "twoshot_ll"])
def test_bf16_parameters_gather_matches_oracle(W, algo):
    """bf16 parameters: the B2_BF16 gather path on the gradient tensors autograd produced, every explicit algorithm."""
    d0 = _check_ddp_against_twins(W, lambda: _ragged_mlp(0).to(torch.bfloat16), oracle.B2O_BF16, algo=algo,
                                  bucket_cap_mb=0.01, first_bucket_mb=0.001)
    assert len(d0.buckets) >= 2 and d0.gathered_buckets > 0 and d0.copied_in_buckets == 0


def test_bucket_of_more_than_max_segments_falls_back_to_copy_in():
    """65 Linear(8, 8) = 130 parameters in ONE bucket: more than a segment table holds, so the bucket is copied in and
    reduced in place - still bit for bit the oracle."""

    def deep():
        torch.manual_seed(0)
        return nn.Sequential(nn.Linear(64, 8), *[nn.Linear(8, 8) for _ in range(64)]).cuda()

    d0 = _check_ddp_against_twins(2, deep, oracle.B2O_F32_WIRE_BF16)
    assert len(d0.buckets) == 1 and len(d0.buckets[0].params) == 130 > 128
    assert d0.copied_in_buckets > 0 and d0.gathered_buckets == 0


def test_state_dict_is_module_prefixed_like_torch_ddp_and_backward_failure_recovers():
    from torchx_b200.ddp import Communicator, DistributedDataParallel

    class Boom(torch.autograd.Function):
        @staticmethod
        def forward(ctx, t):
            return t.clone()

        @staticmethod
        def backward(ctx, g):
            raise RuntimeError("boom")

    class Mid(nn.Module):
        boom = False

        def forward(self, t):
            return Boom.apply(t) if self.boom else t

    def net():
        torch.manual_seed(0)
        return nn.Sequential(nn.Linear(64, 32), nn.ReLU(), Mid(), nn.Linear(32, 8)).cuda()

    comm = Communicator.create(0, 1, 0, "/unused")
    try:
        d = DistributedDataParallel(net(), comm, bucket_cap_mb=0.001, first_bucket_mb=0.0005)
        keys = list(d.state_dict().keys())
        assert keys and all(k.startswith("module.") for k in keys)  # what torch DDP checkpoints look like
        d.load_state_dict(d.state_dict())
        x = torch.randn(4, 64, device="cuda")
        d.module[2].boom = True
        with pytest.raises(RuntimeError, match="boom"):
            # the last layer's gradients are counted in, then backward dies: the engine drops the queued callback
            d(x).square().mean().backward()
        d.module[2].boom = False
        d.zero_grad(set_to_none=True)
        d(x).square().mean().backward()  # the next iteration starts from clean reducer state
        torch.cuda.synchronize()
        twin = net()
        twin(x).square().mean().backward()
        want = oracle.allreduce(oracle.B2O_F32_WIRE_BF16, [_flat_grads(twin)], 1.0)
        assert_bits_equal(_flat_grads(d.module), want, "after a failed backward")
    finally:
        comm.close()
