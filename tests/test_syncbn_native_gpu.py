"""SyncBatchNorm on the native BatchNorm2d kernels, on the GPU: every output, gradient, running statistic and
num_batches_tracked bit-equal to the ATen-compute path the layer took before (``_FabricSyncBatchNorm``, and F.batch_norm
at one rank), with W ranks sharing one device through worker processes (tests/workers/syncbn_native_worker.py)."""
import os
import subprocess
import sys
import uuid

import copy

import numpy as np
import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_workers(tmp_path, world, mode, timeout=300):
    shm = f"/b2_sbnn_{uuid.uuid4().hex[:12]}"
    procs, logs = [], [tmp_path / f"{mode}{world}_{r}.log" for r in range(world)]
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "syncbn_native_worker.py"), "--rank", str(r), "--world",
               str(world), "--device", "0", "--shm", shm, "--mode", mode, "--out", str(tmp_path / f"{mode}{world}_{r}.npz")]
        with open(logs[r], "w") as f:
            procs.append(subprocess.Popen(cmd, stdout=f, stderr=subprocess.STDOUT))
    try:
        for p in procs:
            p.wait(timeout=timeout)
    except subprocess.TimeoutExpired:
        pass
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    failed = [f"rank {r} exited with {p.returncode}:\n{logs[r].read_text()[-6000:]}" for r, p in enumerate(procs) if p.returncode != 0]
    assert not failed, "\n".join(failed)
    return [dict(np.load(tmp_path / f"{mode}{world}_{r}.npz")) for r in range(world)]


def assert_bit_equal(res):
    """No mismatch between the native and the ATen-compute run on any rank, and every rank ran as many collectives."""
    for r, got in enumerate(res):
        assert str(got["bad"]) == "", f"rank {r}: differ from the ATen-compute path:\n{got['bad']}"
    assert len({int(got["op_count"]) for got in res}) == 1, [int(got["op_count"]) for got in res]


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_layers_bit_equal_to_the_aten_path(tmp_path, world):
    """ResNet-50's 12 BatchNorm shapes with unequal per-rank batches, momentum None, no running statistics, eps = 0 with
    zero-variance channels, and +-0 / NaN / +-inf inputs with outputs that round to +-0, two steps each; at W = 1 against
    F.batch_norm.  Then a native forward + backward with no host sync (sync debug mode "error")."""
    res = run_workers(tmp_path, world, "layers")
    assert_bit_equal(res)
    for got in res:
        assert int(got["native"]) >= 2 * (15 if world == 1 else 16)  # every case's layer took the native path in both steps
        assert int(got["nosync.native"]) == 1


def test_mixed_paths_in_one_step(tmp_path):
    """Rank 0 NCHW, rank 1 an empty batch, rank 2 a misaligned view, rank 3 native, in one step: two layers back to back
    and a fused Bottleneck whose bn3 and downsample BatchNorm are both 64 wide, bit-equal to the ATen-compute path with
    every op counter equal at the end."""
    res = run_workers(tmp_path, 4, "mixed")
    assert_bit_equal(res)
    assert int(res[1]["native"]) == 0 and int(res[3]["native"]) > 0


def test_fused_block_whose_batchnorm_input_needs_no_gradient(tmp_path):
    """W = 2: a fused BasicBlock with conv1 frozen and an input that needs no gradient, so bn1's input needs none while its
    weight is trainable.  NCHW fp32 (ATen's compute inside the fused block, whose general backward reduce forms no sums
    without input_g) and channels-last bf16 (native), bit-equal to the unfused ATen-compute path."""
    res = run_workers(tmp_path, 2, "frozen")
    assert_bit_equal(res)
    assert all(int(got["native"]) > 0 for got in res)


def _misaligned_like(t):
    """A channels-last view of t's values whose data pointer is 2 bytes past a 16-byte boundary."""
    n, c, h, w = t.shape
    buf = torch.empty(t.numel() + 8, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(n, h, w, c).permute(0, 3, 1, 2)
    v.copy_(t)
    assert v.is_contiguous(memory_format=torch.channels_last) and v.data_ptr() % 16 != 0
    return v


@pytest.mark.parametrize("relu", [False, True])
def test_batchnorm2d_takes_a_misaligned_gradient(relu):
    """BatchNorm2d's native backward (and the fused ReLU's) given a channels-last gradient that is not 16-byte aligned:
    the bits of nn.BatchNorm2d (+ relu)."""
    from torchx_b200.nn import BatchNorm2d

    torch.manual_seed(0)
    ref = nn.BatchNorm2d(64).cuda()
    with torch.no_grad():
        ref.weight.uniform_(0.5, 1.5)
        ref.bias.uniform_(-1, 1)
    mine = copy.deepcopy(ref)
    mine.__class__ = BatchNorm2d
    x0 = torch.randn(4, 64, 9, 9, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    go = _misaligned_like(torch.randn(4, 64, 9, 9, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
    grads = []
    for m, fused in ((ref, False), (mine, True)):
        x = x0.clone().requires_grad_()
        if relu:
            out = m.normalise(m.batch_stats(x), relu=True) if fused else torch.relu(m(x))
        else:
            out = m(x)
        out.backward(go)
        grads.append([out, x.grad, m.weight.grad, m.bias.grad])
    for a, b in zip(*grads):
        assert torch.equal(a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32),
                           b.contiguous().view(torch.int16 if b.element_size() == 2 else torch.int32))


@pytest.mark.parametrize("world", [2, 4])
def test_resnets_under_the_mini_ddp(tmp_path, world):
    """resnet50 and resnet18 converted to SyncBatchNorm, 3 SGD steps under the mini-DDP: losses, parameters, gradients and
    buffers bit-equal to the unfused ATen-compute path; in the fused step no ATen BatchNorm, ReLU or threshold_backward
    kernel runs."""
    res = run_workers(tmp_path, world, "nets")
    assert_bit_equal(res)
    for got in res:
        for arch in ("resnet50", "resnet18"):
            assert int(got[f"{arch}.kernels.native_bn"]) > 0
            for k in ("aten_bn", "relu", "threshold"):
                assert int(got[f"{arch}.kernels.{k}"]) == 0, (arch, k)


def test_groups_equal_a_world_of_two(tmp_path):
    """SyncBatchNorm(process_group=B200Group) in two groups of 2 of a W = 4 world: each group rank's results are those of
    the same rank of a W = 2 world."""
    pair = run_workers(tmp_path, 2, "pair")
    groups = run_workers(tmp_path, 4, "groups")
    assert_bit_equal(pair)
    for got in groups:
        assert str(got["bad"]) == ""
    keys = [k for k in pair[0] if k.startswith("pair_")]
    assert keys
    for r, got in enumerate(groups):
        for k in keys:
            assert got[k].tobytes() == pair[r % 2][k].tobytes(), f"rank {r} {k}"
