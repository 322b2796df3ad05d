"""CPU-side checks of the stream-plumbing ABI: the Python enums of b2s_combine_op / b2s_split_op number their members
from 0 (tests/test_abi_mirrors.py holds the header's values to ``_lib``'s); argument validation that needs no device."""
import ctypes as C

import futuresdr_b200 as fb
from futuresdr_b200 import _lib


def test_stream_enums_count_from_zero():
    assert [int(o) for o in fb.CombineOp] == list(range(7))
    assert [int(o) for o in fb.SplitOp] == [0, 1]


def test_stream_calls_validate_before_touching_a_device():
    c, p = C.c_size_t(7), C.c_size_t(7)
    lib = _lib.lib
    # NULL context / out-pointers
    assert lib.b2s_combine_exec(None, 0, None, 0, None, 0, None, 0, C.byref(c), C.byref(p)) == _lib.EINVAL
    assert lib.b2s_split_exec(None, 0, None, 0, None, None, 0, C.byref(c), C.byref(p)) == _lib.EINVAL
    assert lib.b2s_fanout_exec(None, 0, 4, None, 0, None, 1, 0, C.byref(c), C.byref(p)) == _lib.EINVAL
