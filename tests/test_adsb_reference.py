"""CPU checks of the ADS-B oracle (tests/adsb_oracle.c): the CRC on public DF17 frames and against a table-driven
CRC-24, agreement with the numpy transcription, tags that do not depend on how the detector's calls slice the stream,
and the detector's edge rules (resume at t0 + 31, the skip after a failed power check, repeated indices, the
g + 480 < D cut-off, non-finite comparisons), with the hand-worked cases of tests/golden/adsb_known_answers.json."""
import json
import os

import numpy as np
import pytest

import adsb_oracle as orc

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "adsb_known_answers.json")))


@pytest.mark.parametrize("frame", GOLDEN["crc_pass"])
def test_crc_public_frames_and_single_bit_flips(frame):
    bits = orc.hex_to_bits(frame)
    assert orc.check_crc(bits) and orc.crc24_table(bits) == 0
    for k in range(112):
        b = bits.copy()
        b[k] ^= 1
        assert not orc.check_crc(b)


def test_crc_agrees_with_table_crc24():
    rng = np.random.default_rng(3)
    for i in range(10_000):
        bits = rng.integers(0, 2, 112).astype(np.uint8)
        if i % 2:                                           # half of them made valid
            data = orc.bits_to_bytes(np.concatenate([bits[:88], np.zeros(24, np.uint8)]))
            crc = orc.crc24_table(np.unpackbits(np.frombuffer(data, np.uint8)))
            bits[88:] = np.unpackbits(np.frombuffer(crc.to_bytes(3, "big"), np.uint8))
        assert orc.check_crc(bits) == (orc.crc24_table(bits) == 0)


def _stream(n, density, seed, thr=10.0):
    rng = np.random.default_rng(seed)
    s = rng.exponential(1.0, n).astype(np.float32)
    nf = rng.uniform(0.25, 2.0, n).astype(np.float32)
    f = np.where(rng.random(n) < density, rng.uniform(1.01, 4.0, n), rng.uniform(0.0, 0.99, n)).astype(np.float32)
    return s, nf, (np.float32(thr) * nf * f).astype(np.float32)


@pytest.mark.parametrize("density", [0.0, 0.01, 0.5, 1.0])
def test_oracle_matches_numpy(density):
    s, nf, corr = _stream(6000, density, 17)
    s[::97] = np.nan
    nf[::89] = 0.0
    corr[::83] = np.inf
    assert orc.detect(10.0, s, nf, corr) == orc.np_detect(10.0, s, nf, corr)
    for g in range(0, 5000, 37):
        assert np.array_equal(orc.demod_bits(s, g), orc.np_demod_bits(s, g))


@pytest.mark.parametrize("density", [0.01, 0.5, 1.0])
def test_tags_do_not_depend_on_call_slicing(density):
    s, nf, corr = _stream(12_000, density, 23)
    ref = orc.replay(10.0, s, nf, corr)
    rng = np.random.default_rng(24)
    for _ in range(30):
        cuts = np.sort(rng.integers(0, 12_000, rng.integers(1, 60))).tolist()
        assert orc.replay(10.0, s, nf, corr, cuts) == ref
    assert orc.replay(10.0, s, nf, corr, list(range(0, 3000))) == ref


def _case(c):
    n = c["n"]
    s = np.full(n, np.float32(c.get("s", 0.0)), np.float32)
    nf = np.ones(n, np.float32)
    corr = np.zeros(n, np.float32)
    for k, v in c.get("corr", {}).items():
        corr[int(k)] = v
    for k, v in c.get("samples", {}).items():
        s[int(k)] = v
    for k, v in c.get("nf", {}).items():
        nf[int(k)] = v
    return s, nf, corr


@pytest.mark.parametrize("case", GOLDEN["detector"], ids=[c["name"] for c in GOLDEN["detector"]])
def test_hand_worked_detector_cases(case):
    s, nf, corr = _case(case)
    nr, tags = orc.detect(case["threshold"], s, nf, corr)
    assert nr == case["num_read"]
    assert [t[0] for t in tags] == case["tags"]
    assert orc.np_detect(case["threshold"], s, nf, corr)[0] == nr
    _, packets, d = orc.replay(case["threshold"], s, nf, corr)
    assert d == nr
    assert [p[0] for p in packets] == case["demodulated"]


def test_non_finite_comparisons():
    # NaN compares false: no trigger at a NaN corr or a NaN product; inf corr with finite nf triggers; nf = 0 gives
    # a ratio of +-inf or NaN, and corr > thr * 0 triggers for any positive corr
    n = 200
    s, nf, corr = np.ones(n, np.float32), np.ones(n, np.float32), np.zeros(n, np.float32)
    corr[3], corr[40], nf[80], corr[80], nf[120], corr[120] = np.nan, np.inf, 0.0, 1.0, np.nan, 50.0
    got = orc.detect(10.0, s, nf, corr)
    assert got == orc.np_detect(10.0, s, nf, corr)
    assert got[0] == 136                                   # triggers at 40 and 80 skip to 71 and 111
