"""CPU checks of the keyfob receiver's oracle (tests/keyfob_oracle.c) against an independent pure-Python transcription
of decoder.rs, the hand-worked cases of tests/golden/keyfob_known_answers.json, and firdes.lowpass against a numpy
float64 evaluation of basic.rs:25-42."""
import json
import os

import numpy as np
import pytest

import keyfob_oracle as ko


def _pulses(widths, start=0):
    level, out = start, []
    for w in widths:
        out.append(np.full(int(w), level, np.uint8))
        level ^= 1
    return np.concatenate(out)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_python_on_random_0_to_3(seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 4, int(rng.integers(0, 50_000))).astype(np.uint8)
    assert ko.decode(x) == ko.py_decode(x)


def test_oracle_matches_python_on_range_edge_widths():
    rng = np.random.default_rng(7)
    x = _pulses(rng.choice([62, 63, 83, 84, 130, 131, 161, 162, 3, 400], 20_000))
    assert ko.decode(x) == ko.py_decode(x)
    # the same widths around strings that carry a preamble
    rng2 = np.random.default_rng(70)
    y = np.concatenate([np.concatenate([_pulses(rng.choice([62, 63, 83, 84, 130, 131, 161, 162], 40)),
                                        ko.levels_for("10101111" + "".join(rng2.choice(["0", "1"], 9)), rng2, 200)])
                        for _ in range(30)])
    want = ko.py_decode(y)
    assert len(want) >= 30
    assert ko.decode(y) == want


def test_oracle_strings_labels_and_strip():
    rng = np.random.default_rng(8)
    for body, text in [("10101111" + "11010101", "1010111111010101 (Close)"),
                       ("10101111" + "11100011", "1010111111100011 (Open)"),
                       ("10101111" + "10111001", "1010111110111001 (Trunk)"),
                       ("011" + "10101111" + "0101", "101011110101"),
                       ("1010101111" + "10101111", "1010111110101111"),       # overlapping, first occurrence wins
                       ("10101111", "10101111")]:
        x = ko.levels_for(body, rng, lead=300)
        got = ko.decode(x)
        assert got == ko.py_decode(x) and [ko.code_text(c) for c in got] == [text]
    for body in ["", "1010111", "0" * 40, "1101010111"]:                   # no preamble, or fewer than 8 bits
        assert ko.decode(ko.levels_for(body, rng, lead=300)) == []


def test_oracle_long_string_keeps_256_bits_and_true_label():
    rng = np.random.default_rng(9)
    body = "10101111" + "".join(rng.choice(["0", "1"], 400)) + "11100011"
    got = ko.decode(ko.levels_for(body, rng, lead=300))
    assert len(got) == 1 and got[0][1] == len(body) and got[0][2] == 2
    assert ko.code_text(got[0]) == body[:256] + " (Open)"


def test_oracle_any_slicing():
    rng = np.random.default_rng(10)
    x = np.concatenate([ko.levels_for("10101111" + "".join(rng.choice(["0", "1"], 30)), rng, lead=200)
                        for _ in range(20)])
    want = ko.py_decode(x)
    assert len(want) == 20
    for cuts in [[], list(range(1, x.size)), np.cumsum(rng.integers(1, 500, 200)).tolist()]:
        assert ko.decode(x, cuts) == want


def test_oracle_avg_and_slicer_are_f32_literal():
    x = np.random.default_rng(11).standard_normal(10_000).astype(np.float32)
    cur, alpha, alpha_inv, y = np.float32(0), np.float32(0.0001), np.float32(1) - np.float32(0.0001), []
    for v in x:
        cur = np.float32(np.float32(cur * alpha_inv) + np.float32(v * alpha))
        y.append(np.float32(v - cur))
    assert np.array_equal(np.array(y, np.float32).view(np.uint32), ko.Avg().work(x).view(np.uint32))
    s = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45, -1e-45, 2.0], np.float32)
    assert ko.slice_u8(s).tolist() == [0, 0, 0, 1, 0, 1, 0, 1]


def _golden():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "keyfob_known_answers.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", _golden()["decoder"], ids=lambda c: c["name"])
def test_known_answers_on_the_oracle(case):
    x = np.array([int(c) for c in case["items"]], np.uint8)
    want = [[i, t] for i, t in case["codes"]]
    assert [[c[0], ko.code_text(c)] for c in ko.decode(x, case["cuts"])] == want
    assert [[c[0], ko.code_text(c)] for c in ko.py_decode(x)] == want


def _np_lowpass(cutoff, window):
    w = np.asarray(window, np.float64)
    omega_c = 2.0 * np.pi * cutoff
    alpha = (w.size - 1) / 2.0
    out = []
    for n, tap in enumerate(w):
        x = n - alpha
        out.append(tap * (omega_c / np.pi if x == 0.0 else np.sin(omega_c * x) / (np.pi * x)))
    return np.array(out, np.float64).astype(np.float32)


@pytest.mark.parametrize("cutoff", [15e3 / 250e3, 0.25, 0.01, -0.1, 0.49999])
@pytest.mark.parametrize("n", [1, 2, 31, 64, 127, 128])
def test_firdes_lowpass_matches_numpy(cutoff, n):
    from futuresdr_b200 import firdes, windows
    for w in (windows.hamming(n, False), np.ones(n), np.random.default_rng(n).uniform(0, 1, n)):
        assert np.array_equal(firdes.lowpass(cutoff, w).view(np.uint32), _np_lowpass(cutoff, w).view(np.uint32))


def test_firdes_lowpass_refusals_and_keyfob_taps():
    import ctypes as C

    from futuresdr_b200 import firdes, keyfob, windows
    from futuresdr_b200._lib import lib
    for c in (0.5, -0.5, 0.7, float("nan")):
        if c == c:
            with pytest.raises(AssertionError):
                firdes.lowpass(c, np.ones(5))
        assert lib.b2s_firdes_lowpass(c, np.ones(5).ctypes.data_as(C.POINTER(C.c_double)), 5, None, 0) == 0
    assert lib.b2s_firdes_lowpass(0.1, None, 0, None, 0) == 0
    assert lib.b2s_firdes_lowpass(0.1, None, 7, None, 0) == 7
    t = keyfob.lowpass_taps()
    assert t.size == 128 and np.array_equal(t, _np_lowpass(0.06, windows.hamming(128, False)))


def test_code_string_of_a_record():
    from futuresdr_b200 import keyfob
    from futuresdr_b200.blocks import KEYFOB_CODE
    r = np.zeros(1, KEYFOB_CODE)[0]
    r["n_bits"], r["label"] = 16, 1
    r["bits"][:2] = [0xAF, 0xD5]
    assert keyfob.code_string(r) == "1010111111010101 (Close)"
    r["n_bits"] = 300
    assert keyfob.code_string(r).endswith("... (Close)") and len(keyfob.code_string(r)) == 256 + 3 + 8
