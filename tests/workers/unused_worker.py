"""One rank of the find_unused_parameters parity check (spawned by tests/test_unused_params_gpu.py): the mini-DDP with
find_unused_parameters=True against stock torch.nn.parallel.DistributedDataParallel(find_unused_parameters=True) on the
same model, inputs and optimizer.  wire="bf16" is compared with stock DDP running the project's b200_bf16_compress_hook,
wire="f32" with stock DDP's default allreduce (gloo: at W = 2 both divide by 2 exactly and add once).

The model has a channels-last conv trunk, a head each rank skips on different steps (locally unused, globally used), a
head only a no_sync micro-batch uses, 140 small parameters that share a bucket with the first head (more parameters than
a segment table holds: the copy-in path), and a head no rank ever uses, which forms a bucket of its own."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
from torch import nn  # noqa: E402

STEPS = 5


class Net(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.trunk = nn.Conv2d(3, 8, 3)
        self.head_b = nn.Linear(288, 16)  # only the no_sync micro-batch uses it
        self.head_a = nn.Linear(288, 16)  # each rank skips it on different steps
        self.many = nn.ParameterList([nn.Parameter(torch.randn(16) * 0.1) for _ in range(140)])
        self.dead = nn.Linear(40, 40)  # no rank ever uses it

    def forward(self, x, use_a, use_b):
        h = self.trunk(x).relu().flatten(1)
        # weighted so that each parameter's gradient is a slice of a real tensor: a plain sum would hand every one of them
        # the same stride-0 expanded gradient, which autograd may store as one shared .grad for all of them
        mix = torch.linspace(0.5, 1.5, len(self.many), device=x.device).view(-1, 1)
        y = (torch.stack(list(self.many)) * mix).sum(0).expand(x.shape[0], 16)
        if use_a:
            y = y + self.head_a(h)
        if use_b:
            y = y + self.head_b(h)
        return {"y": y, "aux": [(h.mean(),)]}


def loss_of(out):
    return out["y"].square().mean() + 0.1 * out["aux"][0][0]


def use_a(rank, step):
    return step < STEPS - 1 and (step + rank) % 2 == 1  # the last step: no rank uses it


def make_net(device):
    return Net().to(device).to(memory_format=torch.channels_last)


def train(ddp, module, opt, rank, device, snapshots):
    dead0 = [p.detach().clone() for p in module.dead.parameters()]
    for step in range(STEPS):
        opt.zero_grad(set_to_none=(step != 2))
        g = torch.Generator(device=device).manual_seed(100 * step + rank)
        if step % 2 == 1:  # a no_sync micro-batch that uses head_b, which the synced one skips
            xb = torch.randn(4, 3, 8, 8, device=device, generator=g).contiguous(memory_format=torch.channels_last)
            with ddp.no_sync():
                loss_of(ddp(xb, use_a(rank, step), True)).backward()
        x = torch.randn(4, 3, 8, 8, device=device, generator=g).contiguous(memory_format=torch.channels_last)
        loss_of(ddp(x, use_a(rank, step), False)).backward()
        torch.cuda.synchronize()
        snapshots.append({n: (None if p.grad is None else p.grad.detach().cpu().clone()) for n, p in module.named_parameters()})
        opt.step()
    for p, p0 in zip(module.dead.parameters(), dead0):
        assert p.grad is None, "a parameter no rank used got a gradient"
        assert torch.equal(p.detach(), p0), "the optimizer moved a parameter no rank used"
    return {n: p.detach().cpu().clone() for n, p in module.named_parameters()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--shm", required=True)
    ap.add_argument("--port", type=int, required=True)
    a = ap.parse_args()

    from torch.nn.parallel import DistributedDataParallel as TorchDDP

    from torchx_b200.ddp import B200HookState, Communicator, DistributedDataParallel, b200_bf16_compress_hook
    from torchx_b200.ddp import _native as N

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{a.port}", rank=a.rank, world_size=a.world)
    comm = Communicator.create(a.rank, a.world, 0, a.shm, stage_mb=8, timeout_s=60)
    comm.set_timeout(30.0)
    comm.set_max_ctas(8)
    report = []
    optims = {"bf16": lambda ps: torch.optim.SGD(ps, lr=0.05, momentum=0.9, weight_decay=0.01),
              "f32": lambda ps: torch.optim.AdamW(ps, lr=1e-2, weight_decay=0.05)}
    for wire, make_opt in optims.items():
        ref_net = make_net(device)
        ref = TorchDDP(ref_net, find_unused_parameters=True)
        if wire == "bf16":
            ref.register_comm_hook(B200HookState(comm), b200_bf16_compress_hook)
        ref_snaps = []
        ref_params = train(ref, ref_net, make_opt(ref_net.parameters()), a.rank, device, ref_snaps)
        for zero_copy in (True, False):
            net = make_net(device)
            mini = DistributedDataParallel(net, comm, wire=wire, bucket_cap_mb=10240 / 2**20, first_bucket_mb=5120 / 2**20,
                                           zero_copy=zero_copy, find_unused_parameters=True)
            names = {id(p): n for n, p in net.named_parameters()}
            layout = [sorted(names[id(p)].split(".")[0] for p in b.params) for b in mini.buckets]
            assert layout[0] == ["dead", "dead"], layout  # a bucket of only unused parameters
            assert len(mini.buckets[1].params) > N.B2_MAX_SEGMENTS, len(mini.buckets[1].params)  # copy-in
            snaps = []
            params = train(mini, net, make_opt(net.parameters()), a.rank, device, snaps)
            tag = f"wire={wire} zero_copy={zero_copy}"
            for step, (got, want) in enumerate(zip(snaps, ref_snaps)):
                none_got = sorted(n for n, g in got.items() if g is None)
                none_want = sorted(n for n, g in want.items() if g is None)
                assert none_got == none_want, (tag, step, none_got, none_want)
                for n, g in got.items():
                    if g is not None:
                        assert torch.equal(g.contiguous().view(torch.int32), want[n].contiguous().view(torch.int32)), (tag, step, n)
            for n, p in params.items():
                assert torch.equal(p.contiguous().view(torch.int32), ref_params[n].contiguous().view(torch.int32)), (tag, "param", n)
            report.append(f"{tag}: gathered {mini.gathered_buckets} copied {mini.copied_in_buckets}, "
                          f"None at the last step {sorted(n for n, g in snaps[-1].items() if g is None)}")
            if zero_copy:
                assert mini.gathered_buckets > 0 and mini.copied_in_buckets > 0, (mini.gathered_buckets, mini.copied_in_buckets)
            else:
                assert mini.gathered_buckets == 0
    comm.check()
    dist.barrier()
    comm.close()
    dist.destroy_process_group()
    print("\n".join(report))
    print(f"rank {a.rank} ok", flush=True)


if __name__ == "__main__":
    main()
