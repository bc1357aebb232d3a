"""find_unused_parameters without a GPU: the output walk and the autograd graph walk on CPU graphs, the zero segment's
table validation in the C ABI, the constructor keyword and the ZeRO overlap refusal."""
import ctypes
import dataclasses
import inspect

import pytest
import torch
from torch import nn

from torchx_b200.ddp import _native as N
from torchx_b200.ddp import zero as Z
from torchx_b200.ddp.ddp import DistributedDataParallel, _find_tensors, _reached_leaves


@dataclasses.dataclass
class _Out:
    logits: torch.Tensor
    extra: dict
    note: str = "not a tensor"


def test_find_tensors_walks_nested_outputs():
    a, b, c, d = (torch.zeros(1) for _ in range(4))
    out = (a, [b, {"k": c, "s": "x", "n": None}], _Out(d, {"deep": (a,)}), 3)
    assert [id(t) for t in _find_tensors(out)] == [id(a), id(b), id(c), id(d), id(a)]
    assert _find_tensors("text") == [] and _find_tensors(None) == []
    assert _find_tensors(_Out) == []  # a dataclass type, not an instance


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.shared = nn.Linear(4, 4)
        self.viewed = nn.Parameter(torch.randn(16))
        self.branch = nn.Linear(4, 4)
        self.frozen = nn.Linear(4, 4)
        self.frozen.requires_grad_(False)
        self.tail = nn.Linear(4, 2)

    def forward(self, x, use_branch):
        h = self.shared(self.shared(x))  # used twice
        h = h + self.viewed.view(4, 4)[0]  # reached only through a view
        h = self.frozen(h)
        if use_branch:
            h = self.branch(h)
        return {"out": _Out(self.tail(h), {"aux": [h.sum()]})}


def _names(m, ids):
    return sorted(n for n, p in m.named_parameters() if id(p) in ids)


def test_graph_walk_finds_the_parameters_the_output_reaches():
    torch.manual_seed(0)
    m = _Net()
    x = torch.randn(3, 4)
    every = _names(m, _reached_leaves(_find_tensors(m(x, True))))
    assert every == ["branch.bias", "branch.weight", "shared.bias", "shared.weight", "tail.bias", "tail.weight", "viewed"]
    skipped = _names(m, _reached_leaves(_find_tensors(m(x, False))))
    assert skipped == ["shared.bias", "shared.weight", "tail.bias", "tail.weight", "viewed"]
    # only the aux output: the tail is not reached
    out = m(x, True)
    assert _names(m, _reached_leaves(_find_tensors(out["out"].extra))) == [
        "branch.bias", "branch.weight", "shared.bias", "shared.weight", "viewed"]
    with torch.no_grad():
        assert _reached_leaves(_find_tensors(m(x, True))) == set()


def test_graph_walk_counts_an_output_that_is_a_parameter():
    p = nn.Parameter(torch.zeros(2))
    assert _reached_leaves([p, torch.zeros(1)]) == {id(p)}


def test_zero_segment_passes_table_validation_and_null_still_fails():
    L = N.lib()
    segs = (N.B2Segment * 3)()
    segs[0].src, segs[0].begin, segs[0].end = 4096, 0, 10
    segs[1].src, segs[1].begin, segs[1].end = N.B2_SEGMENT_ZEROS, 10, 11
    segs[2].src, segs[2].begin, segs[2].end = N.B2_SEGMENT_ZEROS, 11, 20
    # the table is accepted: the call fails on the next check, the missing communicator
    assert L.b2_allreduce_gather(None, ctypes.c_void_p(4096), 20, segs, 3, 0, 1.0, 0, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"null communicator"
    all_zero = (N.B2Segment * 1)()
    all_zero[0].src, all_zero[0].begin, all_zero[0].end = N.B2_SEGMENT_ZEROS, 0, 20
    assert L.b2_allreduce_gather(None, ctypes.c_void_p(4096), 20, all_zero, 1, 0, 1.0, 0, None) == N.B2_EINVAL
    assert L.b2_last_error() == b"null communicator"
    segs[1].src = None
    assert L.b2_allreduce_gather(None, ctypes.c_void_p(4096), 20, segs, 3, 0, 1.0, 0, None) == N.B2_EINVAL
    assert b"segment 1 does not continue the bucket at element 10" in L.b2_last_error()


def test_header_defines_the_zero_segment_marker():
    import os
    import re

    src = open(os.path.join(os.path.dirname(N.INCLUDE_DIR), "include", "b200ddp.h")).read()
    m = re.search(r"#define\s+B2_SEGMENT_ZEROS\s+\(\(const void\s*\*\)\s*(\d+)\)", src)
    assert m and int(m.group(1)) == N.B2_SEGMENT_ZEROS


def test_constructor_keyword_defaults_to_off():
    p = inspect.signature(DistributedDataParallel.__init__).parameters["find_unused_parameters"]
    assert p.default is False and p.kind is inspect.Parameter.POSITIONAL_OR_KEYWORD


def _stand_in(find_unused):
    """A DistributedDataParallel that was never constructed (no communicator, no GPU): only what the ZeRO constructor
    reads before it refuses."""
    m = DistributedDataParallel.__new__(DistributedDataParallel)
    m.__dict__["find_unused_parameters"] = find_unused
    return m


def test_zero_refuses_overlap_with_find_unused_parameters():
    p = nn.Parameter(torch.zeros(3))
    for cls in (torch.optim.SGD, torch.optim.AdamW):
        with pytest.raises(ValueError, match="overlap_with_ddp=True cannot be combined with find_unused_parameters=True"):
            Z.ZeroRedundancyOptimizer(_stand_in(True), cls, params=[p], overlap_with_ddp=True, lr=0.1)
    # without overlap the constructor goes on (and fails later, on the stand-in's missing state)
    with pytest.raises(AttributeError):
        Z.ZeroRedundancyOptimizer(_stand_in(True), torch.optim.SGD, params=[p], lr=0.1)
    with pytest.raises(AttributeError):
        Z.ZeroRedundancyOptimizer(_stand_in(False), torch.optim.SGD, params=[p], overlap_with_ddp=True, lr=0.1)
