"""dist.init_process_group("b200") on the GPU: W processes sharing one H100, no gloo and no NCCL.  Every dist.* call, stock
DDP (no hook, torch's bf16_compress_hook, b200_bf16_compress_hook), torch.nn.SyncBatchNorm, torch's ZeroRedundancyOptimizer
and the mini-DDP next to group collectives, bit for bit against the oracles (tests/workers/torch_backend_worker.py)."""
import os
import socket
import subprocess
import sys
import uuid

import numpy as np
import pytest
import torch

import oracle
from tests import _exact_oracle as X
from tests._util import assert_bits_equal
from tests.test_exact_ops_gpu import assert_float_sum_equal, float_sum_oracle

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "workers"))
import torch_backend_worker as TW  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run_workers(tmp_path, world, devices):
    shm, port = f"/b2_tpg_{uuid.uuid4().hex[:12]}", _free_port()
    procs = []
    for r in range(world):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "workers", "torch_backend_worker.py"), "--rank", str(r), "--world",
               str(world), "--device", str(devices[r]), "--shm", shm, "--port", str(port), "--out", str(tmp_path / f"r{r}.npz")]
        procs.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            o, _ = p.communicate(timeout=900)
            outs.append(o)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, p in enumerate(procs):
        assert p.returncode == 0, f"rank {r} failed:\n{outs[r]}"
    return [dict(np.load(tmp_path / f"r{r}.npz")) for r in range(world)]


def _inputs(dtype, W, seed):
    return [TW.bits(TW.reduce_input(dtype, r, seed)) for r in range(W)]


def check_collectives(res, W, tag):
    for k, (dtype, ops) in enumerate(TW.OPS.items()):
        for j, op in enumerate(ops):
            xs = _inputs(dtype, W, 10 * k + j)
            what = f"{tag} all_reduce {dtype} {op} W={W}"
            for r in range(W):
                got = res[r][f"{tag}.allreduce.{dtype}.{op}"]
                if W == 1:
                    assert np.array_equal(got, xs[0]), what
                elif op in ("sum", "avg") and X.is_float(dtype):
                    assert_float_sum_equal(dtype, got, float_sum_oracle(dtype, xs, 1.0 if op == "sum" else 1.0 / W), what)
                else:
                    X.assert_exact_equal(dtype, got, X.reduce(dtype, op, xs), what)
    gathered = np.concatenate([np.arange(7, dtype=np.int32) + 100 * r for r in range(W)])
    rs_in = [x[: W * 100] for x in _inputs("float32", W, 77)]
    rs_want = float_sum_oracle("float32", rs_in, 1.0) if W > 1 else rs_in[0]
    rl_want = X.reduce("int64", "max", [x[: W * 50] for x in _inputs("int64", W, 78)])
    rows = [[(i + 2 * j) % 3 for j in range(W)] for i in range(W)]
    for r in range(W):
        g = res[r]
        assert np.array_equal(g[f"{tag}.all_gather_into_tensor"], gathered)
        assert np.array_equal(g[f"{tag}.all_gather"].reshape(-1), gathered)
        assert_float_sum_equal("float32", g[f"{tag}.reduce_scatter_tensor"], rs_want[r * 100:(r + 1) * 100], f"{tag} rs r={r}")
        assert np.array_equal(g[f"{tag}.reduce_scatter"], rl_want[r * 50:(r + 1) * 50])
        for root in range(W):
            assert np.array_equal(g[f"{tag}.broadcast.{root}"].view(np.float32), np.full(33, root * 10 + root, np.float32))
            if r == root:
                want = X.reduce("int64", "sum", _inputs("int64", W, 90 + root))
                assert np.array_equal(g[f"{tag}.reduce.{root}"], want), (tag, root)
            else:  # a non-root rank's tensor is only read
                assert np.array_equal(g[f"{tag}.reduce.{root}"], _inputs("int64", W, 90 + root)[r])
        want = np.concatenate([np.full((rows[i][r], 3), 1000 * i + r, np.int32) for i in range(W)]).reshape(-1, 3)
        assert np.array_equal(g[f"{tag}.all_to_all_single"].reshape(-1, 3), want), (tag, r)
        a2a = g[f"{tag}.all_to_all"].view(np.float32).reshape(-1)
        assert np.array_equal(a2a, np.concatenate([np.full(j + 1, 100 * j + r, np.float32) for j in range(W)])), (tag, r)
        for root in (0, W - 1):
            if r == root:
                assert np.array_equal(g[f"{tag}.gather.{root}"].view(np.float32), np.repeat(np.arange(W, dtype=np.float32)[:, None], 5, 1))
            assert np.array_equal(g[f"{tag}.scatter.{root}"].view(np.float32), np.full(5, 10 * root + r, np.float32))
        if tag == "async":
            assert (g[f"{tag}.reuse_after_async"] == -7).all()
        if W > 1:
            prv = (r - 1) % W
            ring = g[f"{tag}.ring"]
            assert np.array_equal(ring, np.arange(ring.size, dtype=np.int32) + prv), (tag, r)
            assert np.array_equal(g[f"{tag}.sendrecv"].view(np.float32), np.full(9, prv, np.float32))


def _bf16_hook_oracle(locals_, W):
    """torch's bf16_compress_hook over this group: bf16(g) * (1/W) rounded to bf16 on each rank, the rank-order bf16 allreduce
    SUM, widened back to fp32."""
    inv = np.float32(1.0) / np.float32(W)  # ATen divides a CUDA tensor by a scalar as a product with its reciprocal
    c = [TW.bits(torch.from_numpy(g).to(torch.bfloat16).float().mul_(float(inv)).to(torch.bfloat16)) for g in locals_]
    s = oracle.allreduce(oracle.B2O_BF16, c, 1.0) if W > 1 else c[0]
    return torch.from_numpy(s.view(np.int16).copy()).view(torch.bfloat16).float().numpy()


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_torch_backend_one_device(tmp_path, world):
    res = run_workers(tmp_path, world, [0] * world)
    W = world
    # 1. dist.*, blocking and async
    for tag in ("sync", "async"):
        check_collectives(res, W, tag)
    for r in range(W):
        g = res[r]
        assert g["obj.all_gather"].tolist() == [q * 1000 + q * 37 for q in range(W)]
        assert g["obj.broadcast"].all()
        assert g["obj.scatter"].tolist() == [r * r]
        assert g["helper.allreduce"].tolist() == [W - 1] * 5
    assert res[0]["obj.gather"].tolist() == list(range(W))
    # 2. stock DDP
    for name in ("mlp", "conv"):
        locals_ = [g[f"ddp.{name}.local"] for g in res]
        div = [(x * (np.float32(1.0) / np.float32(W))).astype(np.float32) for x in locals_]  # the Reducer's div_ on the GPU
        want = {"none": oracle.allreduce(oracle.B2O_F32, div, 1.0) if W > 1 else div[0],
                "torch_bf16": _bf16_hook_oracle(locals_, W),
                "b200_bf16": oracle.allreduce(oracle.B2O_F32_WIRE_BF16, locals_, 1.0 / W)}
        for hook, wv in want.items():
            for r in range(W):
                assert_bits_equal(res[r][f"ddp.{name}.{hook}.grads"], wv, f"stock DDP {name} {hook} rank {r}")
                assert res[r][f"ddp.{name}.{hook}.params"].tobytes() == res[0][f"ddp.{name}.{hook}.params"].tobytes()
                if name == "mlp":
                    assert not res[r][f"ddp.{name}.{hook}.marker_after_init"].any()  # rank 0's buffer after construction
                    assert not res[r][f"ddp.{name}.{hook}.marker"].any()  # ... and after each forward
    # 3. torch.nn.SyncBatchNorm under the group == this package's SyncBatchNorm on the fabric
    keys = [k[len("sbn_fabric."):] for k in res[0] if k.startswith("sbn_fabric.")]
    assert len(keys) >= 6 * 4
    for r in range(W):
        for k in keys:
            assert res[r]["sbn_torch." + k].tobytes() == res[r]["sbn_fabric." + k].tobytes(), f"rank {r} SyncBatchNorm {k}"
    # 4. torch's ZeroRedundancyOptimizer == the unsharded optimizer, both over stock DDP on the group
    for r in range(W):
        assert res[r]["zero.zero"].tobytes() == res[r]["zero.plain"].tobytes(), f"rank {r} ZeRO parameters"
        assert res[r]["zero.zero"].tobytes() == res[0]["zero.zero"].tobytes()
    assert res[0]["zero.consolidated_steps"].tolist() == [3.0] * 6
    # 5. the mini-DDP next to group collectives: gradients, the collectives around it and the op counts
    locals_ = [g["mini.local"] for g in res]
    want = oracle.allreduce(oracle.B2O_F32, locals_, 1.0 / W)
    for r in range(W):
        g = res[r]
        assert_bits_equal(g["mini.grads"], want, f"mini-DDP gradients rank {r}")
        assert np.array_equal(g["mini.pending"].view(np.float32), np.full(1000, sum(range(W)), np.float32))
        for step in range(2):
            assert np.array_equal(g[f"mini.a1.{step}"].view(np.float32), np.full(3, sum(q + step for q in range(W)), np.float32))
            assert np.array_equal(g[f"mini.a2.{step}"].view(np.float32), np.full(3, W - 1, np.float32))
        assert np.array_equal(g["mini.async_forward.allreduce"].view(np.float32), np.full(1024, W * (W + 1) / 2, np.float32))
        assert g["mini.async_forward.nbt"].tolist() == (6 if W > 1 else 10 * r + 6)
        if W > 1:  # the backward's buckets, torch SyncBatchNorm's backward allreduce, then the dist.all_reduce after it
            assert g["mini.op_counts"].tolist() == [int(g["mini.buckets"]) + 2] * 2, g["mini.op_counts"]
    # 7. capture is refused before anything reaches the communicator
    for r in range(W):
        assert res[r]["capture.refused"].tolist() == [True, True, True]
        assert int(res[r]["capture.op_delta"]) == 0
    # 6. destroy and re-init on the same communicator
    for r in range(W):
        assert np.array_equal(res[r]["reinit.allreduce"].view(np.float32), np.full(4, W * (W + 1) / 2, np.float32))


@pytest.mark.parametrize("world", [2, 4])
def test_torch_backend_across_devices(tmp_path, world, cuda_count):
    if cuda_count < world:
        pytest.skip(f"needs {world} GPUs")
    res = run_workers(tmp_path, world, list(range(world)))
    check_collectives(res, world, "sync")
    check_collectives(res, world, "async")


def test_example_trains_under_local_cuda(tmp_path, cuda_count):
    """examples/train_stock_ddp.py through the local_cuda scheduler at 1x2: identical parameters on both ranks."""
    if cuda_count < 2:
        pytest.skip("needs 2 GPUs")
    env = dict(os.environ, PYTHONPATH=ROOT, TRAIN_STOCK_DDP_OUT=str(tmp_path))
    cmd = [sys.executable, "-m", "torchx_b200.cli.main", "run", "-s", "local_cuda", "dist.ddp", "-j", "1x2", "--script",
           os.path.join(ROOT, "examples", "train_stock_ddp.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout
    got = [torch.load(tmp_path / f"params{r}.pt") for r in range(2)]
    for a, b in zip(got[0], got[1]):
        assert torch.equal(a, b)
