"""The Python mirrors of include/b200sdr.h agree with what a C compiler makes of the header: every struct the library
fills for Python has the size and field offsets of its numpy dtype or ctypes Structure, and every constant has its
``_lib`` value.  A Rust bindgen / cgo binding sees exactly these numbers.  One probe program prints them all."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from futuresdr_b200 import _lib, blocks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

STRUCTS = [
    ("b2s_handshake", _lib.Handshake),
    ("b2s_adsb_packet", blocks.ADSB_PACKET),
    ("b2s_adsb_detection", blocks.ADSB_DETECTION),
    ("b2s_zigbee_frame", blocks.ZIGBEE_FRAME),
    ("b2s_keyfob_code", blocks.KEYFOB_CODE),
]

# header name B2S_<n> -> _lib.<n>
_MIRRORED = """OK EINVAL ECUDA ENOMEM EAGAIN EUNSUPPORTED ESTATE ETIMEOUT
INSUFFICIENT_INPUT INSUFFICIENT_OUTPUT BOTH_SUFFICIENT
F32_F32 C32_F32 C32_C32 F64_F64
ALGO_AUTO ALGO_DIRECT ALGO_TENSOR ALGO_FFT ALGO_SCAN
OP_SCALE_F32 OP_SCALE_C32 OP_QUAD_DEMOD OP_NORM_SQR OP_QUAD_DEMOD_C32 OP_EXP_F32 OP_MAG_C32 OP_LOG10_F32
OP_DC_BLOCK_F32 OP_SLICE_F32_U8
WAVE_COS WAVE_SIN WAVE_SQUARE
COMBINE_ADD_F32 COMBINE_SUB_F32 COMBINE_MUL_F32 COMBINE_CONJ_MUL_C32 COMBINE_MAG_DIV_C32_F32 COMBINE_TO_C32
COMBINE_TO_C32_NEG_Q
SPLIT_RE_IM SPLIT_DUP_F32
KEYFOB_NONE KEYFOB_CLOSE KEYFOB_OPEN KEYFOB_TRUNK""".split()
CONSTANTS = [("B2S_" + n, getattr(_lib, n)) for n in _MIRRORED] + [("B2S_IPC_HANDLE_BYTES", 64)]


def _layout(mirror):
    """(size, {field: offset}) of a numpy structured dtype or a ctypes Structure."""
    if isinstance(mirror, np.dtype):
        return mirror.itemsize, {f: mirror.fields[f][1] for f in mirror.names}
    return C.sizeof(mirror), {f: getattr(mirror, f).offset for f, *_ in mirror._fields_}


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    """{"sizeof <struct>" | "<struct>.<field>" | "<constant>": value} as the C compiler sees the header."""
    lines = []
    for struct, mirror in STRUCTS:
        lines.append(f'printf("sizeof {struct} %zu\\n", sizeof({struct}));')
        lines += [f'printf("{struct}.{f} %zu\\n", offsetof({struct}, {f}));' for f in _layout(mirror)[1]]
    lines += [f'printf("{name} %lld\\n", (long long)({name}));' for name, _ in CONSTANTS]
    tmp = tmp_path_factory.mktemp("abi_probe")
    src, exe = tmp / "probe.c", tmp / "probe"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200sdr.h"\nint main(void) {\n    '
                   + "\n    ".join(lines) + "\n    return 0;\n}\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    return {key: int(value) for key, value in (line.rsplit(" ", 1) for line in out.splitlines())}


@pytest.mark.parametrize("struct,mirror", STRUCTS, ids=[s for s, _ in STRUCTS])
def test_struct_layout(probe, struct, mirror):
    size, offsets = _layout(mirror)
    assert probe[f"sizeof {struct}"] == size
    assert {f: probe[f"{struct}.{f}"] for f in offsets} == offsets


@pytest.mark.parametrize("name,value", CONSTANTS, ids=[n for n, _ in CONSTANTS])
def test_constant(probe, name, value):
    assert probe[name] == value


def test_algo_scan_keeps_its_number():
    # the IIR's scan algorithm was added to b2s_algo as 4, after the FIR algorithms; its number does not change
    assert _lib.ALGO_SCAN == 4
