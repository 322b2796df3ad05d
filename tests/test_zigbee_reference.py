"""CPU checks of the ZigBee oracle (tests/zigbee_oracle.c) that the device blocks are compared against: agreement with
an independent numpy float32 transcription, the Mac's CRC-16 against a table-driven one and on every single-bit flip
of Mac-framed frames, the same results under many call slicings, and the hand-worked known answers of
tests/golden/zigbee_known_answers.json."""
import json
import os

import numpy as np
import pytest

import zigbee_oracle as zo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "zigbee_known_answers.json")
MM = (2.0, 0.000225, 0.5, 0.03, 0.0002)


def _eq(a, b):
    """bit for bit, except that any NaN equals any NaN (payloads and signs of NaN differ between libraries)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def _phase_like(n, seed):
    rng = np.random.default_rng(seed)
    return (np.sin(np.arange(n) * 0.7) * 1.2 + 0.3 * rng.standard_normal(n)).astype(np.float32)


def _chips(rng, n_frames):
    parts, frames = [], []
    for s in range(n_frames):
        parts.append(rng.integers(0, 2, int(rng.integers(0, 800))).astype(np.uint8))
        f = zo.mac_frame(rng.integers(0, 256, int(rng.integers(1, 100))).astype(np.uint8).tobytes(), s)
        frames.append(f[5:])
        parts.append(zo.chips_of(f))
    c = np.concatenate(parts + [np.zeros(40, np.uint8)])
    return np.where(c > 0, 1.0, -1.0).astype(np.float32), frames


def test_dc_block_matches_numpy():
    x = _phase_like(5000, 1)
    x[[7, 99]] = [np.inf, np.nan]
    for alpha in (0.00016, 0.5, 1.0):
        y, _ = zo.np_dc_block(alpha, x)
        assert _eq(zo.DcBlock(alpha).work(x), y)


@pytest.mark.parametrize("params", [MM, (2.0, 0.01, 0.2, 0.2, 0.05), (1.0, 0.0, 0.0, 0.0, 0.0), (0.5, 0.001, 0.9, 0.6, 0.0)])
def test_mm_matches_numpy(params):
    x = _phase_like(6000, 2)
    for n_out in (10, 100_000):
        c, o, e = zo.np_mm(params, x, n_out)
        c2, o2, e2 = zo.Mm(*params).work(x, n_out)
        assert (c, e) == (c2, e2) and _eq(o, o2)


def test_decoder_matches_numpy():
    rng = np.random.default_rng(3)
    x, frames = _chips(rng, 12)
    noisy = x.copy()
    noisy[rng.integers(0, x.size, x.size // 40)] *= -1
    for s in (x, noisy, rng.standard_normal(20_000).astype(np.float32)):
        for thr in (3, 6, 10):
            assert zo.Decoder(thr).work(s) == zo.np_decode(thr, s)
    assert [b for _, b in zo.Decoder(6).work(x)] == frames


def test_crc_against_table_on_random_frames():
    rng = np.random.default_rng(4)
    for _ in range(10_000):
        d = rng.integers(0, 256, int(rng.integers(0, 128))).astype(np.uint8).tobytes()
        assert zo.calc_crc(d) == zo.crc16_table(d)


def test_crc_on_every_single_bit_flip_of_mac_frames():
    rng = np.random.default_rng(5)
    for s in range(6):
        body = zo.mac_frame(rng.integers(0, 256, int(rng.integers(1, 40))).astype(np.uint8).tobytes(), s)[5:]
        assert zo.crc_ok(body)
        for k in range(8 * len(body)):
            b = bytearray(body)
            b[k // 8] ^= 1 << (k % 8)
            assert zo.calc_crc(bytes(b)) != 0
    assert not zo.crc_ok(b"\x00\x00") and zo.calc_crc(b"") == 0


def test_slicing_does_not_change_results():
    rng = np.random.default_rng(6)
    x = _phase_like(30_000, 7)
    whole, pos, err = zo.mm_replay(MM, x)
    for cuts in ([1, 2, 3, 4, 5], np.cumsum(rng.integers(1, 2000, 20)).tolist(), [29_990]):
        o, p, e = zo.mm_replay(MM, x, cuts)
        assert (p, e) == (pos, err) and np.array_equal(o.view(np.uint32), whole.view(np.uint32))
        o, p, e = zo.mm_replay(MM, x, cuts, n_out=333)
        assert (p, e) == (pos, err) and np.array_equal(o.view(np.uint32), whole.view(np.uint32))
    dc = zo.DcBlock(0.00016).work(x)
    blk = zo.DcBlock(0.00016)
    assert np.array_equal(np.concatenate([blk.work(x[a:b]) for a, b in [(0, 1), (1, 777), (777, 30_000)]]).view(
        np.uint32), dc.view(np.uint32))
    c, _ = _chips(rng, 20)
    ref = zo.decode_replay(6, c)
    for cuts in (range(1, 3000), np.cumsum(rng.integers(1, 500, 60)).tolist(), [32, 64, 65]):
        assert zo.decode_replay(6, c, list(cuts)) == ref


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", _golden()["decoder"], ids=lambda c: c["name"])
def test_known_answers_decoder(case):
    x = np.array([1.0 if ch == "1" else -1.0 for ch in case["chips"]], np.float32)
    want = [(i, bytes.fromhex(h)) for i, h in case["frames"]]
    assert zo.decode_replay(case["threshold"], x, case.get("cuts")) == want
    assert zo.np_decode(case["threshold"], x) == want


@pytest.mark.parametrize("case", _golden()["mm"], ids=lambda c: c["name"])
def test_known_answers_mm(case):
    x = np.array([float(v) for v in case["input"]], np.float32)
    m = zo.Mm(*case["params"])
    c, o, err = m.work(x, case["n_out"])
    assert c == case["consumed"] and err == case["err"]
    assert _eq(o, np.array(case["outputs_bits"], np.uint32).view(np.float32))
    assert int(np.float32(m.s.omega).view(np.uint32)) == case["omega_after_bits"]
    if case["name"] == "mu_exactly_integral":
        assert np.array_equal(o, x[:o.size])
    if case["name"].startswith("clamp"):
        lim = np.float32(np.float32(case["params"][0]) * np.float32(case["params"][4]))
        mid = np.float32(case["params"][0])
        assert np.float32(m.s.omega) in (mid + lim, mid - lim)
