"""The ZigBee transmitter's CPU oracle (tests/zigbee_tx_oracle.c) against an independent numpy transcription and the
reference's literal DSSS table and SHAPE (tests/golden/zigbee_tx_dsss.json); the Mac's drop and sequence rules; the
burst_start tags; the library's host helpers; and the oracle's stream back through the receiver oracle (QuadDemod, DC
blocker, ClockRecoveryMm, Decoder of rx.rs), every frame decoded.  Apart from the table this parity is unpinned: the
reference's ZigBee code has no transmitter tests.  No GPU needed."""
import os
import subprocess

import numpy as np
import pytest

from futuresdr_b200 import _lib, blocks, zigbee

import zigbee_oracle as zo
import zigbee_tx_oracle as zt

HERE = os.path.dirname(os.path.abspath(__file__))
MM = (zigbee.MM_OMEGA, zigbee.MM_GAIN_OMEGA, zigbee.MM_MU, zigbee.MM_GAIN_MU, zigbee.MM_OMEGA_RELATIVE_LIMIT)


def _pays(rng, lengths):
    return [rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in lengths]


def test_generated_dsss_table_and_shape_are_the_reference_literals():
    fx = zt.golden()
    assert "modulator.rs" in fx["source"]
    want = np.array(fx["dsss"], np.float32)
    assert want.shape == (16, 16, 2) and np.all(np.abs(want) == 1)
    assert np.array_equal(zt.dsss().view(np.uint32), want.view(np.uint32))
    assert np.array_equal(zt.shape().view(np.uint32), np.array(fx["shape"], np.float32).view(np.uint32))
    assert np.float32(fx["shape"][1]) == np.float32(np.sqrt(0.5))
    # rows 0 and 8 are the IEEE 802.15.4 chip sequences of symbols 0 and 8, chip 2c on I and 2c + 1 on Q
    for nib, seq in ((0, "11011001110000110101001000101110"), (8, "10001100100101100000011101111011")):
        chips = np.stack([want[nib, :, 0], want[nib, :, 1]], axis=1).reshape(-1) > 0
        assert "".join("1" if c else "0" for c in chips) == seq


@pytest.mark.parametrize("pad", [0, 1, 40000])
def test_oracle_matches_the_transcription(pad):
    """Payloads of every length 0-116 in one push, through the C chain under several buffer and output capacities."""
    rng = np.random.default_rng(pad)
    lengths = list(range(0, 117)) if pad < 40000 else list(range(0, 117, 9)) + [116]
    rng.shuffle(lengths)
    pays = _pays(rng, lengths)
    want, wb = zt.np_stream(pays, pad)
    assert [b[1] for b in wb] == [zt.frame_len(len(p), pad) for p in pays]
    for c1, c2, caps in ((4096, 1 << 16, [1 << 22]), (1, 1, [4096]), (7, 333, [1, 7, 4096]),
                         (16, 5000, [int(c) for c in rng.integers(1, 50000, 40)])):
        if caps == [1, 7, 4096] and pad == 40000:
            caps = [7, 4096, 100_003]
        t = zt.Tx(pad, c1, c2)
        assert t.push(*pays) == 0
        got, bursts = t.stream(caps)
        assert zt.same_bits(got, want), (c1, c2, caps)
        assert bursts == wb


def test_sequence_number_wraps_past_255():
    rng = np.random.default_rng(5)
    pays = _pays(rng, rng.integers(0, 30, 300))
    t = zt.Tx(1)
    assert t.push(*pays) == 0
    got, bursts = t.stream([1 << 20])
    want, wb = zt.np_stream(pays, 1)
    assert zt.same_bits(got, want) and bursts == wb
    # frames 0 and 256 carry the same sequence number, 255 and 256 differ
    f = [zo.mac_frame(p, s) for s, p in enumerate(pays)]
    assert f[256][7] == 0 and f[255][7] == 255


def test_oversized_payload_is_dropped_without_a_sequence_number():
    rng = np.random.default_rng(6)
    a, big, edge, b = _pays(rng, [10, 117, 116, 3])
    t = zt.Tx(0)
    assert t.push(a, big, edge, b) == 1
    got, bursts = t.stream([1 << 20])
    want = np.concatenate([zt.np_frame(zo.mac_frame(p, s), 0) for s, p in enumerate([a, edge, b])])
    assert zt.same_bits(got, want)
    assert [n for _, n in bursts] == [zt.frame_len(n, 0) for n in (10, 116, 3)]


def test_bursts_sit_on_each_front_pad():
    rng = np.random.default_rng(7)
    pays = _pays(rng, [0, 116, 50])
    t = zt.Tx(40000, 64, 1000)
    t.push(*pays)
    got, bursts = t.stream([30_001])
    idx = 0
    for (i, n), p in zip(bursts, pays):
        assert i == idx and n == 2 * 40000 + 128 * (len(p) + 16) + 2 == zigbee.frame_len(len(p))
        assert not got[i:i + 40000].view(np.uint32).any()              # +0.0 pads
        assert not got[i + n - 40000:i + n].view(np.uint32).any()
        idx += n
    assert idx == got.size and zigbee.frame_len(116) == 96_898


def test_sign_of_zero_and_the_q_delay():
    """Every fourth modulator sample is a chip times SHAPE[0] = 0.0: -0.0 for a negative chip.  Q is two samples late:
    +0.0 leads it, and the two held Q values, beside I = +0.0, close the body."""
    p = b"\x00\xff\x5a"
    t = zt.Tx(3)
    t.push(p)
    x, _ = t.stream()
    body = x[3:-3]
    assert body.size == 128 * len(zo.mac_frame(p, 0)) + 2
    re, im = body.real, body.imag
    for z in (re[:-2:4], im[2::4]):
        assert np.all(z == 0) and np.signbit(z).any() and not np.signbit(z).all()
    assert np.all(re[1:-2:4] != 0) and np.all(im[3::4] != 0)
    for z in (im[:2], re[-2:]):
        assert np.all(z == 0) and not np.signbit(z).any()
    h = np.float32(np.sqrt(0.5))                                     # the last chip's Q at SHAPE[1], SHAPE[2], SHAPE[3]
    assert np.array_equal(np.abs(im[-3:]), np.array([h, 1.0, h], np.float32))


def test_loopback_through_the_receiver_oracle():
    """The oracle's stream (pad 40000) through numpy QuadDemod and the receiver oracle with rx.rs's parameters decodes
    every frame, in order and with a good FCS, as the Mac framed it."""
    rng = np.random.default_rng(8)
    pays = _pays(rng, rng.integers(0, 117, 20))
    t = zt.Tx()
    t.push(*pays)
    x, _ = t.stream([1 << 22])
    xd = x.astype(np.complex128)
    last = np.concatenate([[0], xd[:-1]])
    phase = np.angle(np.conj(last) * xd).astype(np.float32)               # QuadDemod: (last.conj() * i).arg()
    dc = zo.DcBlock(zigbee.DC_ALPHA).work(phase)
    mm, _, err = zo.mm_replay(MM, dc)
    assert err is None
    got = zo.decode_replay(zigbee.DECODER_THRESHOLD, mm)
    assert [by for _, by in got] == [zo.mac_frame(p, s)[5:] for s, p in enumerate(pays)]
    assert all(zo.crc_ok(by) for _, by in got)


def test_host_helpers():
    assert zigbee.PADDING == _lib.ZIGBEE_PADDING == zt.PADDING
    assert zigbee.MAX_PAYLOAD == _lib.ZIGBEE_MAX_PAYLOAD == zt.MAX_PAYLOAD
    for n in (0, 1, 116):
        for pad in (0, 1, 40000):
            assert zigbee.frame_len(n, pad) == zt.frame_len(n, pad)


def test_header_mirror_of_the_new_constants(tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200sdr.h"\nint main(void) {\n'
                   '    printf("%d %d %zu %zu %zu\\n", B2S_ZIGBEE_MAX_PAYLOAD, B2S_ZIGBEE_PADDING,\n'
                   '           sizeof(b2s_zigbee_burst), offsetof(b2s_zigbee_burst, index), offsetof(b2s_zigbee_burst, len));\n'
                   '    return 0;\n}\n')
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-I", os.path.join(os.path.dirname(HERE), "include"), str(src), "-o",
                    str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    d = blocks.ZIGBEE_BURST
    assert got == [_lib.ZIGBEE_MAX_PAYLOAD, _lib.ZIGBEE_PADDING, d.itemsize, d.fields["index"][1], d.fields["len"][1]]
