"""reduce and the six object collectives of torchx_b200.distributed in two processes sharing one GPU: the same worker
(tests/workers/reduce_objects_worker.py) under init_pg("b200") and under a 2-rank gloo process group on CPU tensors,
where every call is torch.distributed's own, must produce the same results (for reduce: on the root; gloo also writes a
non-root's tensor, which the fabric only reads)."""
import math

import numpy as np
import pytest

from tests.test_reduce_gpu import _run_workers
from tests.test_reduce_scatter_gpu import _free_port

pytestmark = pytest.mark.gpu


def test_b200_equals_gloo_two_processes_one_gpu(tmp_path):
    fabric = _run_workers(tmp_path, 2, [0, 0], "b200")
    gloo = _run_workers(tmp_path, 2, [0, 0], "gloo", port=_free_port())
    for r in range(2):
        only_fabric = {"reduce_float32_max_nan", "reduce_bf16_avg"}
        assert set(fabric[r]) - set(gloo[r]) == only_fabric, sorted(fabric[r])
        for k, want in gloo[r].items():
            if k.startswith("reduce_") and r != 1:  # gloo's reduce uses a non-root's tensor as scratch; ours only reads it
                continue
            assert fabric[r][k] == want, (r, k)
    f32 = [float(np.float32(x)) for x in (0.1, -1.5, 3e38, 0.0)]
    assert fabric[0]["reduce_int32_min"] == ("torch.int32", [5, 0, 2**31 - 1, -(2**31)])
    assert fabric[0]["reduce_float32_sum"] == ("torch.float32", f32)

    # what gloo cannot check: float MAX with a NaN and signed zeros, and bf16 AVG, on root 1
    _, m = fabric[1]["reduce_float32_max_nan"]
    assert m[0] == 1.0 and math.isnan(m[1]) and m[2] == 0.0 and math.copysign(1, m[2]) == 1 and m[3] == -1.0
    assert fabric[1]["reduce_bf16_avg"] == ("torch.bfloat16", [1.5, 4.5, -0.375])
    _, m0 = fabric[0]["reduce_float32_max_nan"]  # rank 0's tensor is only read
    assert m0[:2] == [0.0, 0.0] and math.copysign(1, m0[1]) == -1 and m0[3] == -1.0
    assert fabric[0]["reduce_bf16_avg"] == ("torch.bfloat16", [1.0, 3.0, -0.25])

    # the results themselves, beyond agreeing with gloo
    assert fabric[1]["reduce_int64_sum"] == ("torch.int64", [3, -3 - 3 + 10, (1 << 63) - 2**64 + 1, -(1 << 63)])
    assert fabric[0]["reduce_int64_sum"] == ("torch.int64", [1, -3, 1 << 62, -(1 << 62)])
    for r in range(2):
        g = fabric[r]
        assert [o["rank"] for o in g["all_gather_object"]] == [0, 1]
        assert g["all_gather_object"][1]["nested"]["t"] == ("torch.int64", "cpu", [1, 2, 3])
        assert g["broadcast_object_list"][2]["cuda"] == ("torch.float32", "cuda", [7.0, 7.0])
        assert g["scatter_object_list"][0] == ({"to": 0, "big": g["scatter_object_list"][0]["big"]} if r == 0 else [None, ()])
    assert fabric[0]["gather_object"] is None and [o["from"] for o in fabric[1]["gather_object"]] == [0, 1]
    assert len(fabric[1]["gather_object"][0]["big"]) == 5 << 20
    assert fabric[1]["recv_object_list_src"] == 0 and fabric[0]["recv_object_list_src"] == 1
    assert fabric[1]["recv_object_list"][1]["cuda"] == ("torch.int64", "cuda", [0, 1, 2, 3])
    assert fabric[0]["recv_object_list"] == [[]]
