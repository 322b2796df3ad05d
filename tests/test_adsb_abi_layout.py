"""The ADS-B ABI structs (b2s_adsb_packet, b2s_adsb_detection in include/b200sdr.h) as a C compiler lays them out must
match the numpy dtypes the Python layer drains them into (blocks.ADSB_PACKET, blocks.ADSB_DETECTION)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_adsb_struct_layouts_match_the_numpy_dtypes(tmp_path):
    from futuresdr_b200.blocks import ADSB_DETECTION, ADSB_PACKET
    probe = tmp_path / "probe.c"
    probe.write_text('''#include <stdio.h>
#include <stddef.h>
#include "b200sdr.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu\\n", sizeof(b2s_adsb_packet), offsetof(b2s_adsb_packet, preamble_index),
           offsetof(b2s_adsb_packet, preamble_correlation), offsetof(b2s_adsb_packet, crc_passed),
           offsetof(b2s_adsb_packet, bytes));
    printf("%zu %zu %zu\\n", sizeof(b2s_adsb_detection), offsetof(b2s_adsb_detection, index),
           offsetof(b2s_adsb_detection, value));
    return 0;
}
''')
    exe = tmp_path / "probe"
    r = subprocess.run(["/usr/bin/gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    f = ADSB_PACKET.fields
    assert [int(v) for v in lines[0].split()] == [ADSB_PACKET.itemsize, f["preamble_index"][1],
                                                  f["preamble_correlation"][1], f["crc_passed"][1], f["bytes"][1]]
    g = ADSB_DETECTION.fields
    assert [int(v) for v in lines[1].split()] == [ADSB_DETECTION.itemsize, g["index"][1], g["value"][1]]
