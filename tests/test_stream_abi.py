"""CPU-side checks of the stream-plumbing ABI: the enum values of b2s_combine_op / b2s_split_op agree between the
header, as a C compiler sees it, and the ctypes mirror; argument validation that needs no device."""
import ctypes as C
import os
import subprocess

import futuresdr_b200 as fb
from futuresdr_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_stream_enums_match_the_header(tmp_path):
    probe = tmp_path / "probe.c"
    probe.write_text('''#include <stdio.h>
#include "b200sdr.h"
int main(void) {
    printf("%d %d %d %d %d %d %d\\n", (int)B2S_COMBINE_ADD_F32, (int)B2S_COMBINE_SUB_F32, (int)B2S_COMBINE_MUL_F32,
           (int)B2S_COMBINE_CONJ_MUL_C32, (int)B2S_COMBINE_MAG_DIV_C32_F32, (int)B2S_COMBINE_TO_C32,
           (int)B2S_COMBINE_TO_C32_NEG_Q);
    printf("%d %d\\n", (int)B2S_SPLIT_RE_IM, (int)B2S_SPLIT_DUP_F32);
    return 0;
}
''')
    exe = tmp_path / "probe"
    r = subprocess.run(["/usr/bin/gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    assert [int(v) for v in lines[0].split()] == [
        _lib.COMBINE_ADD_F32, _lib.COMBINE_SUB_F32, _lib.COMBINE_MUL_F32, _lib.COMBINE_CONJ_MUL_C32,
        _lib.COMBINE_MAG_DIV_C32_F32, _lib.COMBINE_TO_C32, _lib.COMBINE_TO_C32_NEG_Q]
    assert [int(v) for v in lines[1].split()] == [_lib.SPLIT_RE_IM, _lib.SPLIT_DUP_F32]
    assert [int(o) for o in fb.CombineOp] == list(range(7))
    assert [int(o) for o in fb.SplitOp] == [0, 1]


def test_stream_calls_validate_before_touching_a_device():
    c, p = C.c_size_t(7), C.c_size_t(7)
    lib = _lib.lib
    # NULL context / out-pointers
    assert lib.b2s_combine_exec(None, 0, None, 0, None, 0, None, 0, C.byref(c), C.byref(p)) == _lib.EINVAL
    assert lib.b2s_split_exec(None, 0, None, 0, None, None, 0, C.byref(c), C.byref(p)) == _lib.EINVAL
    assert lib.b2s_fanout_exec(None, 0, 4, None, 0, None, 1, 0, C.byref(c), C.byref(p)) == _lib.EINVAL
