"""The op counter's entry points without a GPU: b2_comm_set_param("op_count", v) and b2_comm_op_count refuse what they must
before touching CUDA, and the binding declares b2_comm_op_count with a 64-bit result (tests/test_op_count_gpu.py runs the
collectives at the counts they set)."""
import ctypes
import os

from torchx_b200.ddp import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_binding_signature():
    assert N.SIGNATURES["b2_comm_op_count"] == (ctypes.c_uint64, [ctypes.c_void_p])
    # the value travels as a long long: op counts past 2^32 reach the library whole
    assert N.SIGNATURES["b2_comm_set_param"][1][2] is ctypes.c_longlong


def test_set_param_op_count_argument_checks():
    L = N.lib()
    for value in (0, 1 << 29, 1 << 40, -1):
        assert L.b2_comm_set_param(None, b"op_count", value) == N.B2_EINVAL, value
        assert b"b2_comm_set_param: bad arguments" in L.b2_last_error(), value


def test_op_count_argument_checks():
    L = N.lib()
    L.b2_comm_set_param(None, b"max_ctas", 1)  # some other error first: the message below must be op_count's own
    assert L.b2_comm_op_count(None) == 0
    assert L.b2_last_error() == b"b2_comm_op_count: null communicator"


def test_header_documents_the_knob_beside_the_others():
    src = open(os.path.join(ROOT, "include", "b200ddp.h")).read()
    knobs = src[src.index('"oneshot_max_bytes"'):src.index("int b2_comm_set_param(")]
    assert '"op_count"' in knobs
