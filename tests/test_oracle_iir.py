"""CPU checks of the IirFilter oracle (tests/iir_oracle.py, crates/futuredsp/src/iir.rs:78-178): the reference's own
known-answer vectors, and bit equality with a line-by-line numpy transcription of taps_accessor_work on ragged call
sequences that split the memory fill across calls."""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import iir_oracle as orc  # noqa: E402  (tests/iir_oracle.py)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "reference_iir_known_answers.json")
CASES = json.load(open(FIXTURE))["cases"]


def feed(filter_call, inputs):
    """The Feeder of iir.rs:186-203: append one sample, filter into a one-item slice, drain what was consumed."""
    buf, outs = [], []
    for v in inputs:
        buf.append(v)
        c, p, _st, y = filter_call(np.array(buf), 1)
        assert c == p
        del buf[:c]
        outs.append(float(y[0]) if p else None)
    return outs


class NumpyIir:
    """iir.rs:78-178 transcribed with numpy scalars of the sample type (one rounding per operation)."""

    def __init__(self, a, b, dtype):
        self.T = np.dtype(dtype).type
        self.a = [self.T(v) for v in a]
        self.b = [self.T(v) for v in b]
        self.memory = []

    def filter(self, i, out_cap):
        T, a, b, memory = self.T, self.a, self.b, self.memory
        i = [T(v) for v in i]
        o = []
        empty = 2 if out_cap == 0 else 0
        if not i:
            return 0, 0, empty, o
        num_filled = 0
        while len(memory) < len(a):
            if len(i) <= len(memory):
                return 0, 0, empty, o
            memory.append(i[len(memory)])
            num_filled += 1
        if num_filled == len(i):
            return 0, 0, empty, o
        n_consumed = n_produced = 0
        with np.errstate(all="ignore"):
            while n_consumed + len(b) - 1 < len(i) and n_produced < out_cap:
                y = T(0)
                for j in range(len(b)):
                    y = T(y + T(b[j] * i[n_consumed + len(b) - j - 1]))
                for j in range(len(a)):
                    y = T(y + T(a[j] * memory[j]))
                for j in range(len(memory) - 1, 0, -1):
                    memory[j] = memory[j - 1]
                if memory:
                    memory[0] = y
                o.append(y)
                n_produced += 1
                n_consumed += 1
        if n_consumed == len(i) and n_produced == out_cap:
            st = 2
        elif n_consumed < len(i):
            st = 1
        else:
            st = 0
        return n_consumed, n_produced, st, o


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_oracle_reproduces_reference_vectors(case, dtype):
    f = orc.Iir(case["a"], case["b"], dtype)
    if case["mode"] == "feeder":
        assert feed(f.filter, case["input"]) == case["expected"]
    else:
        c, p, _st, y = f.filter(np.array(case["input"]), case["out_cap"])
        assert (c, p) == (len(case["expected"]),) * 2
        assert y.tolist() == case["expected"]


def ragged_calls(rng, n_a, n_b, total):
    """Call lengths 0, 1, < n_a, < n_b and large, with output capacities that are sometimes short or zero."""
    sizes = [0, 1, max(n_a - 1, 0), max(n_b - 1, 0), 1, 0, int(rng.integers(1, 400)), total]
    return [(s, int(rng.choice([0, 1, s, s + 3, max(s // 2, 1)]))) for s in sizes]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n_a,n_b", [(0, 1), (0, 3), (1, 1), (2, 3), (3, 1), (4, 6), (8, 9)])
def test_oracle_matches_numpy_transcription_on_ragged_calls(dtype, n_a, n_b):
    rng = np.random.default_rng(1000 + 10 * n_a + n_b)
    a = (rng.uniform(-1, 1, n_a) / max(n_a, 1) * 0.9).astype(dtype)
    b = rng.uniform(-1, 1, n_b).astype(dtype)
    x = rng.standard_normal(3000).astype(dtype)
    x[17] = np.finfo(dtype).tiny / 8                         # a denormal sample
    ref, ora = NumpyIir(a, b, dtype), orc.Iir(a, b, dtype)
    pos = 0
    for want, cap in ragged_calls(rng, n_a, n_b, 1500):
        sl = x[pos: pos + want]
        r1 = ref.filter(sl, cap)
        r2 = ora.filter(sl, cap)
        assert r1[:3] == r2[:3], (want, cap, r1[:3], r2[:3])
        np.testing.assert_array_equal(np.array(r1[3], dtype).view(np.uint8), r2[3].view(np.uint8))
        pos += r2[0]


def test_oracle_exact_arbiter_agrees_with_f64_oracle():
    rng = np.random.default_rng(5)
    a = np.float32([1.6, -0.8])
    b = np.float32([0.1, 0.2, 0.1])
    x = rng.standard_normal(5000).astype(np.float32)
    ex = orc.iir_exact(a, b, x)
    y64 = orc.iir(a.astype(np.float64), b.astype(np.float64), x.astype(np.float64), np.float64)
    np.testing.assert_array_equal(ex, y64)
    y32 = orc.iir(a, b, x)
    assert np.max(np.abs(y32 - ex)) < 1e-4
