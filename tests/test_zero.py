"""ZeRO-1 pieces that need no GPU: b2_reduce_scatter_gather's header, binding and host-side checks, the shard arithmetic
(padding, block intersections against a pure-Python restatement) and ZeroRedundancyOptimizer's argument checks."""
import ctypes
import itertools

import pytest
import torch

from torchx_b200.ddp import _native as N
from torchx_b200.ddp import zero as Z


def test_declared_bound_and_exported():
    src = open(N.INCLUDE_DIR + "/b200ddp.h").read()
    assert "int b2_reduce_scatter_gather(b2_comm_t* comm, void* out, size_t block, const b2_segment_t* segments" in src
    assert "b2_reduce_scatter_gather" in N.SYMBOLS
    L = N.lib()
    assert L.b2_reduce_scatter_gather.argtypes[3] is ctypes.POINTER(N.B2Segment)
    assert N.B2_ABI_VERSION == 3 == L.b2_version()


def test_host_checks_in_order():
    L = N.lib()
    segs = (N.B2Segment * 1)()
    segs[0].src, segs[0].begin, segs[0].end = 4096, 0, 16
    # the mode first, then block == 0 (a no-op: nothing else is read), then the communicator
    assert L.b2_reduce_scatter_gather(None, ctypes.c_void_p(4096), 8, segs, 1, 5, 1.0, None) == N.B2_EINVAL
    assert b"b2_reduce_scatter_gather: unknown mode 5" in L.b2_last_error()
    assert L.b2_reduce_scatter_gather(None, ctypes.c_void_p(4096), 0, segs, 1, 7, 1.0, None) == N.B2_EINVAL
    for mode in range(5):
        assert L.b2_reduce_scatter_gather(None, None, 0, None, 0, mode, 1.0, None) == N.B2_OK
        assert L.b2_reduce_scatter_gather(None, ctypes.c_void_p(4096), 8, segs, 1, mode, 1.0, None) == N.B2_EINVAL
        assert b"null communicator" in L.b2_last_error()


def test_allreduce_gather_texts_unchanged_by_the_shared_table_check():
    L = N.lib()
    segs = (N.B2Segment * 2)()
    segs[0].src, segs[0].begin, segs[0].end = 4096, 0, 10
    segs[1].src, segs[1].begin, segs[1].end = 8192, 10, 20
    assert L.b2_allreduce_gather(None, ctypes.c_void_p(4096), 21, segs, 2, 0, 1.0, 0, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"b2_allreduce_gather: segments cover 20 elements, bucket has 21"


@pytest.mark.parametrize("W", range(1, 9))
def test_padded_block(W):
    for n in itertools.chain(range(1, 300), [4095, 4096, (1 << 17) + 3, 6_553_600]):
        B = Z.padded_block(n, W)
        assert B % 8 == 0 and W * B >= n
        assert B - 8 < -(-n // W) <= B  # the smallest vec multiple that holds ceil(n / W)


def _intersections_by_element(offsets, numels, block, rank):
    """Restatement: walk every element of the rank's block and record which parameter holds it."""
    owner = {}
    for i, (o, n) in enumerate(zip(offsets, numels)):
        for e in range(o, o + n):
            owner[e] = i
    out = {}
    for e in range(rank * block, (rank + 1) * block):
        if e in owner:
            i = owner[e]
            lo, hi = out.get(i, (e, e))
            assert hi == e  # contiguous
            out[i] = (lo, e + 1)
    return [(i, lo, hi) for i, (lo, hi) in sorted(out.items())]


@pytest.mark.parametrize("numels", [[1], [7, 9], [3, 1, 100, 8, 8, 17], [64] * 9, [1000, 1, 1, 1, 333]])
@pytest.mark.parametrize("W", [1, 2, 3, 4, 8])
def test_block_intersections_match_restatement(numels, W):
    offsets = [sum(numels[:i]) for i in range(len(numels))]
    B = Z.padded_block(sum(numels), W)
    covered = 0
    for r in range(W):
        got = Z.block_intersections(offsets, numels, B, r)
        assert got == _intersections_by_element(offsets, numels, B, r)
        covered += sum(hi - lo for _, lo, hi in got)
    assert covered == sum(numels)  # every element in exactly one rank's block


class _FakeDDP:
    pass


def test_optimizer_allow_list_and_model_type():
    p = torch.nn.Parameter(torch.zeros(3))
    for cls in (torch.optim.RMSprop, torch.optim.Adagrad, torch.optim.LBFGS, object):
        with pytest.raises(TypeError, match="supports SGD, Adam, AdamW"):
            Z.ZeroRedundancyOptimizer(_FakeDDP(), cls, params=[p], lr=0.1)
    with pytest.raises(TypeError, match="DistributedDataParallel"):
        Z.ZeroRedundancyOptimizer(_FakeDDP(), torch.optim.AdamW, params=[p], lr=0.1)


def test_group_checks():
    a, b, c = (torch.nn.Parameter(torch.zeros(2)) for _ in range(3))
    Z._check_groups(Z._normalize_groups([a, b, c]), [a, b, c])
    Z._check_groups(Z._normalize_groups([{"params": [a]}, {"params": [b, c], "lr": 0.5}]), [a, b, c])
    with pytest.raises(ValueError, match="in no parameter group"):
        Z._check_groups(Z._normalize_groups([a, b]), [a, b, c])
    with pytest.raises(ValueError, match="more than one group"):
        Z._check_groups(Z._normalize_groups([{"params": [a, b]}, {"params": [b, c]}]), [a, b, c])
    with pytest.raises(ValueError, match="not a trainable parameter"):
        Z._check_groups(Z._normalize_groups([a, b, c, torch.nn.Parameter(torch.zeros(1))]), [a, b, c])
    with pytest.raises(ValueError, match="empty parameter list"):
        Z._normalize_groups([])


def test_memory_script_state_bytes_are_exact():
    import importlib.util
    import os

    spec = importlib.util.spec_from_file_location("zero_memory", os.path.join(os.path.dirname(N.INCLUDE_DIR), "tools", "zero_memory.py"))
    zm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(zm)
    m = torch.nn.Sequential(torch.nn.Linear(33, 7), torch.nn.Linear(7, 1))  # 238 + 8 elements, one bucket
    n = 33 * 7 + 7 + 7 + 1
    for W in (1, 2, 4):
        got = zm.state_bytes(m, W)
        assert got["unsharded_state_bytes"] == 8 * n
        B = Z.padded_block(n, W)
        assert got["sharded_state_bytes"] == 8 * min(B, n)  # rank 0's block, the fullest
