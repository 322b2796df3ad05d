"""The WLAN transmitter's CPU oracle (tests/wlan_oracle.c) against an independent Python transcription and the
reference's literal tables (tests/golden/wlan_tables.json), the reference's state rules (stale pad bits, the scrambler
seed and sequence number wraps), the library's host helpers, and the oracle's frames back through a Python
restatement of the receive direction (tests/wlan_model.py).  Apart from the tables this parity is unpinned: the
reference's only WLAN test asserts nothing.  No GPU needed."""
import os
import subprocess
import zlib

import numpy as np
import pytest

from futuresdr_b200 import _lib, blocks, wlan

import wlan_model as wm
import wlan_oracle as wo

HERE = os.path.dirname(os.path.abspath(__file__))


def _pay(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def _c64(pairs) -> np.ndarray:
    return np.array([complex(a, b) for a, b in pairs], np.complex64)


def test_generated_tables_are_the_reference_tables():
    fx = wo.golden()
    sync = _c64(fx["sync_words"])
    assert np.array_equal(wo.sync_words().view(np.uint32), sync.view(np.uint32))
    assert np.array_equal(wo.py_sync_words().view(np.uint32), sync.view(np.uint32))
    assert [1 - 2 * int(b) for b in wo.mseq()] == fx["polarity"]
    assert list(wo.mseq()) == wo.py_mseq()
    assert list(wo.signal_pattern()) == fx["signal_interleaver"]
    for bpsc, name in ((1, "bpsk"), (2, "qpsk"), (4, "qam16"), (6, "qam64")):
        want = _c64(fx["constellation"][name])
        assert np.array_equal(wo.constellation(bpsc).view(np.uint32), want.view(np.uint32)), name
        assert np.array_equal(wo.py_constellation(bpsc).view(np.uint32), want.view(np.uint32)), name


def test_crc_and_frame_param():
    for n in (0, 1, 24, 1524):
        d = _pay(n, n)
        assert wo.crc32(d) == zlib.crc32(d)
    for m in wlan.Mcs:
        for psdu in range(28, 1529, 7):
            bits = 16 + 8 * psdu + 6
            ns = -(-bits // m.n_dbps)
            want = (ns, ns * m.n_dbps, ns * m.n_dbps - bits)
            assert wo.frame_param(m, psdu) == want
            fp = wlan.FrameParam.new(m, psdu)
            assert (fp.n_symbols, fp.n_data_bits, fp.n_pad) == want and fp.mcs == m and fp.psdu_size == psdu
    with pytest.raises(_lib.B200SdrError):
        wlan.FrameParam.new(8, 100)
    with pytest.raises(_lib.B200SdrError):
        wlan.FrameParam.new(0, 1529)


def test_mcs_table():
    assert [m.n_cbps for m in wlan.Mcs] == [48, 48, 96, 96, 192, 192, 288, 288]
    assert [m.n_dbps * 2 // m.n_cbps for m in wlan.Mcs if m != wlan.Mcs.QAM64_2_3] == [1, 1, 1, 1, 1, 1, 1]
    assert wlan.Mcs.QAM64_2_3.n_dbps * 3 == wlan.Mcs.QAM64_2_3.n_cbps * 2
    assert [m.rate_field for m in wlan.Mcs] == list(wo.RATE)
    assert wlan.Mcs.parse("QAM64-3_4") == wlan.Mcs.QAM64_3_4 and wlan.Mcs.parse("bpsk12") == wlan.Mcs.BPSK_1_2
    with pytest.raises(ValueError):
        wlan.Mcs.parse("qam256")


@pytest.mark.parametrize("mcs", range(8))
def test_oracle_matches_the_transcription(mcs):
    """Every PSDU length 28..1528 in steps, in an order that leaves stale pad bits of every kind, through one C and one
    Python transmitter; the mapped symbols and Prefix's samples for a few of them."""
    lengths = list(range(0, 1501, 37)) + [1500, 1499, 0, 1, 2, 3]
    order = np.random.default_rng(mcs).permutation(len(lengths))
    t, pt = wo.Tx(), wo.PyTx()
    for i, k in enumerate(order):
        p = _pay(lengths[k], 100 * mcs + i)
        a, b = t.frame(p, mcs), pt.frame(p, mcs)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), lengths[k]
        if i < 3:
            mp = wo.mapped(a[1], mcs)
            py = np.stack([wo.py_map(s, 1 if j == 0 else wo.N_BPSC[mcs], j) for j, s in enumerate(a[1])])
            assert np.array_equal(mp.view(np.uint32), py.view(np.uint32))
            y = np.stack([wo.ifft_f64(v) for v in mp]).astype(np.complex64)
            for pf, ptl in ((0, 0), (5000, 5000), (3, 1)):
                got = wo.prefix(y, pf, ptl)
                assert got.size == wo.frame_len(len(mp), pf, ptl) == wlan.frame_len(mcs, lengths[k], pf, ptl)
                assert np.array_equal(got.view(np.uint64), wo.py_prefix(y, pf, ptl).view(np.uint64))
    assert t.frame(b"x" * 1501, mcs) is None and pt.frame(b"x" * 1501, mcs) is None


def test_stale_pad_bits_come_from_the_last_longer_frame():
    """encoder.rs never clears `bits`: after a 1500-byte frame A and a 900-byte frame B, a short frame's pad bytes j
    are B's where B is longer than j, else A's.  Its symbols differ from the same frame after other long frames, and
    its PSDU does not."""
    a, b, s = _pay(1500, 1), _pay(900, 2), _pay(100, 3)
    pt = wo.PyTx()
    psdu_a, _ = pt.frame(a, 0)
    psdu_b, _ = pt.frame(b, 0)
    psdu_s, sym_s = pt.frame(s, 0)
    n = len(psdu_s)
    stale = np.packbits(np.array(pt.bits[16:16 + 8 * 1528], np.uint8).reshape(-1, 8)[:, ::-1], axis=1).reshape(-1)
    assert np.array_equal(stale[:n], psdu_s)
    assert np.array_equal(stale[n:len(psdu_b)], psdu_b[n:])
    assert np.array_equal(stale[len(psdu_b):], psdu_a[len(psdu_b):])
    t2 = wo.Tx()
    t2.frame(_pay(1500, 9), 0)
    t2.frame(_pay(900, 8), 0)
    psdu2, sym2 = t2.frame(s, 0)
    assert np.array_equal(psdu2, psdu_s) and not np.array_equal(sym2, sym_s)


def test_seed_and_sequence_number_wrap():
    pt = wo.PyTx()
    for i in range(127):
        pt.frame(b"", 0)
    assert pt.seed == 1 and pt.seq == 127
    t, pt = wo.Tx(seq=4094, seed=126), wo.PyTx(seq=4094, seed=126)
    seqs = []
    for i in range(4):
        a, b = t.frame(b"abc", 2), pt.frame(b"abc", 2)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        seqs.append(int(a[0][22]) | int(a[0][23]) << 8)
    assert seqs == [4094 << 4, 4095 << 4, 0, 1 << 4]
    assert pt.seed == 3                                # 126, 127, 1, 2 used


@pytest.mark.parametrize("mcs", range(8))
def test_every_payload_round_trips_through_the_receive_model(mcs):
    t = wo.Tx()
    frames = [_pay(n, n + mcs) for n in (0, 1, 500, 1500)]
    for p in frames:
        psdu, sym = t.frame(p, mcs)
        y = np.stack([wo.ifft_f64(v) for v in wo.mapped(sym, mcs)]).astype(np.complex64)
        x = wo.prefix(y, 50, 20)
        assert wm.decode_burst(x, 0, 50) == (p, mcs)
        x[50 + 320 + 80 + 40] += 5                      # a symbol hit hard enough: FCS or SIGNAL check fails
        x[50 + 320 + 40] += 5
        r = wm.decode_burst(x, 0, 50)
        assert r is None or r == (p, mcs)


def test_header_mirror_of_the_new_constants(tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200sdr.h"\nint main(void) {\n'
                   '    printf("%d %d %zu %zu %zu %d %d %d %d %d %d %d %d\\n", B2S_WLAN_MAX_PAYLOAD, B2S_WLAN_MAX_PSDU,\n'
                   '           sizeof(b2s_wlan_burst), offsetof(b2s_wlan_burst, index), offsetof(b2s_wlan_burst, len),\n'
                   '           B2S_WLAN_BPSK_1_2, B2S_WLAN_BPSK_3_4, B2S_WLAN_QPSK_1_2, B2S_WLAN_QPSK_3_4,\n'
                   '           B2S_WLAN_QAM16_1_2, B2S_WLAN_QAM16_3_4, B2S_WLAN_QAM64_2_3, B2S_WLAN_QAM64_3_4);\n'
                   '    return 0;\n}\n')
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-I", os.path.join(os.path.dirname(HERE), "include"), str(src), "-o",
                    str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    d = blocks.WLAN_BURST
    assert got == [_lib.WLAN_MAX_PAYLOAD, _lib.WLAN_MAX_PSDU, d.itemsize, d.fields["index"][1], d.fields["len"][1],
                   *[int(m) for m in wlan.Mcs]]
