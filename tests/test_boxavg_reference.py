"""CPU checks of the MovingAverage oracle (tests/boxavg_oracle.c): the reference's own Mocker known answers, agreement
with an independent numpy float32 transcription, and the rules of the work() call loop."""
import json
import os

import numpy as np
import pytest

from boxavg_oracle import MAX_ITER, BoxAvgRef, np_work

CASES = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_boxavg_known_answers.json")))["cases"]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _same(got, want):
    """Bit equality, any NaN matching any NaN (payloads are not part of the contract)."""
    g = np.ascontiguousarray(got).view(np.float32)
    w = np.ascontiguousarray(want).view(np.float32)
    assert g.shape == w.shape
    gn, wn = np.isnan(g), np.isnan(w)
    assert np.array_equal(gn, wn)
    assert np.array_equal(g[~gn].view(np.uint32), w[~wn].view(np.uint32))


@pytest.mark.parametrize("case", CASES, ids=[c["cite"].split()[-1] for c in CASES])
def test_oracle_reproduces_mocker_known_answers(case):
    """Mocker::run: work() while call_again, on a finished input, into `reserve` items."""
    ref = BoxAvgRef(np.float32, case["len"])
    x = np.asarray(case["input"], np.float32)
    c = p = 0
    outs = []
    while True:
        r = ref.work(x[c:], case["reserve"] - p)
        c += r.consumed
        p += r.produced
        outs.append(r.out)
        if not r.call_again:
            break
    assert np.concatenate(outs).tolist() == case["output"], case["cite"]


def test_f32_sum_folds_from_negative_zero():
    """`impl Sum<&f32> for f32` starts at -0.0 in the std the reference builds with: a window of -0.0 sums to -0.0.
    (From +0.0 the first output would be +0.0.)  Complex32 folds from Complex::zero() = (+0, +0)."""
    ref = BoxAvgRef(np.float32, 3)
    ref.pad = 0
    r = ref.work(np.full(3, -0.0, np.float32), 1)
    assert r.produced == 1 and _bits(r.out)[0] == 0x80000000
    cref = BoxAvgRef(np.complex64, 3)
    cref.pad = 0
    r = cref.work(np.full(3, complex(-0.0, -0.0), np.complex64), 1)
    assert r.out.view(np.uint32).tolist() == [0, 0]              # +0 + -0 = +0 in each component
    one = BoxAvgRef(np.float32, 1)                              # len 1: the empty prefix is the fold's start value
    r = one.work(np.asarray([-0.0, -0.0], np.float32), 2)
    assert _bits(r.out).tolist() == [0x80000000, 0]             # -0 + -0 = -0; then (-0 - -0) + -0 = +0


def _values(rng, n, dtype, specials):
    x = rng.standard_normal(n).astype(np.float32)
    if specials:
        pool = np.asarray([0.0, -0.0, 1e-45, -1e-45, 1e-40, np.inf, -np.inf, np.nan, 3e38, -3e38], np.float32)
        k = rng.integers(0, n, max(1, n // 50))
        x[k] = pool[rng.integers(0, pool.size, k.size)]
    if np.dtype(dtype) == np.complex64:
        y = rng.standard_normal(n).astype(np.float32)
        if specials:
            k = rng.integers(0, n, max(1, n // 50))
            y[k] = np.asarray([np.inf, -0.0, np.nan, 1e-42], np.float32)[rng.integers(0, 4, k.size)]
        return (x + 1j * y).astype(np.complex64) if not specials else _cplx(x, y)
    return x


def _cplx(re, im):
    z = np.empty(re.size, np.complex64)
    z.real, z.imag = re, im
    return z


@pytest.mark.parametrize("dtype,length,divisor", [
    (np.float32, 1, None), (np.float32, 2, None), (np.float32, 48, None), (np.float32, 64, None),
    (np.float32, 300, 4800.0), (np.complex64, 1, None), (np.complex64, 3, None), (np.complex64, 48, None),
])
def test_oracle_matches_numpy_transcription(dtype, length, divisor):
    """Random ragged call sequences, with signed zeros, denormals, infinities and NaN in the stream."""
    rng = np.random.default_rng(length * 7 + (dtype == np.complex64))
    n = 9000
    x = _values(rng, n, dtype, True)
    ref = BoxAvgRef(dtype, length, divisor)
    pad, pos = length - 1, 0
    while True:
        n_in = int(min(n - pos, rng.integers(0, 5000)))
        cap = int(rng.integers(0, 4500))
        sl = x[pos:pos + n_in]
        want = np_work(dtype, length, divisor, pad, sl, cap)
        got = ref.work(sl, cap)
        assert (got.consumed, got.produced, got.call_again, got.finished) == want[1:5]
        assert ref.pad == want[0]
        _same(got.out, want[5])
        pad, pos = want[0], pos + got.consumed
        if pos + length > n and pad == 0:
            break


def test_call_loop_rules():
    ref = BoxAvgRef(np.float32, 5)
    x = np.arange(1, 11, dtype=np.float32)
    r = ref.work(x, 0)                                          # capacity 0 in the pad: nothing, no call_again
    assert (r.consumed, r.produced, r.call_again, r.finished, ref.pad) == (0, 0, False, False, 4)
    r = ref.work(x, 3)                                          # pad across calls; m == out_len: no call_again
    assert (r.consumed, r.produced, r.call_again, r.finished, ref.pad) == (0, 3, False, False, 1)
    r = ref.work(x, 3)                                          # the last pad item; m < out_len: call_again
    assert (r.consumed, r.produced, r.call_again, r.finished, ref.pad) == (0, 1, True, False, 0)
    assert r.out.tolist() == [0.0]
    r = ref.work(x[:4], 8)                                      # fewer than len items, input finished: finished
    assert (r.consumed, r.produced, r.call_again, r.finished) == (0, 0, False, True)
    r = ref.work(x[:4], 8, finished=False)
    assert r.finished is False
    r = ref.work(x, 0)                                          # capacity 0 after the pad: m = 0 != 6
    assert (r.consumed, r.produced, r.finished) == (0, 0, False)
    r = ref.work(x, 4)
    assert (r.consumed, r.produced, r.finished) == (4, 4, False)
    assert r.out.tolist() == [15.0, 20.0, 25.0, 30.0]
    r = ref.work(x[4:], 10)                                     # 6 items left: 2 outputs, all of them -> finished
    assert (r.consumed, r.produced, r.finished) == (2, 2, True) and r.out.tolist() == [35.0, 40.0]


def test_runs_are_capped_at_max_iter_and_restart_the_sum():
    """A call covers at most 4000 outputs, and the next call re-folds its prefix: a NaN from inf - inf ends with the
    call that made it."""
    ref = BoxAvgRef(np.float32, 3)
    ref.pad = 0
    x = np.ones(MAX_ITER + 10, np.float32)
    x[MAX_ITER - 2] = np.inf                                    # enters at output 3996, leaves at output 3998
    e = ref.run(x, x.size)
    assert (e.consumed, e.produced, e.calls) == (x.size - 2, x.size - 2, 3)
    assert np.isinf(e.out[MAX_ITER - 4:MAX_ITER - 1]).all()
    assert np.isnan(e.out[MAX_ITER - 1])                        # (inf - inf) + 1: the last output of the first call
    assert (e.out[MAX_ITER:] == 3.0).all()                      # the second call restarts clean from x[4000]


def test_exec_emulation_stops_at_max_calls_and_at_no_progress():
    ref = BoxAvgRef(np.complex64, 4)
    x = np.ones(9000, np.complex64)
    e = ref.run(x, 100, max_calls=1)
    assert (e.consumed, e.produced, e.calls, e.call_again, e.done) == (0, 3, 1, True, False)
    e = ref.run(x, 20_000)
    assert (e.consumed, e.produced, e.calls, e.call_again, e.done) == (8997, 8997, 4, False, True)
