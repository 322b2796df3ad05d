"""CPU cross-check of tests/pfb_exact.py: at every shape and call pattern the GPU tests use, the oracle's outputs land on
the integers the exactness argument promises (the drivers assert it), every call pattern gives the same stream, and
the oracle's steady state equals a float64 textbook restatement of each block."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pfb_exact as px  # noqa: E402


def _chan_stream(calls):
    arms = [out[2] for (_, _, _, (c, p, ca), out) in calls if p]
    return np.concatenate(arms, axis=1) if arms else np.zeros((0, 0))


@pytest.mark.parametrize("N,T,osr,nofused", px.CHAN_SHAPES)
def test_chan_oracle_exact(N, T, osr, nofused):
    rng, taps, D = px.chan_case(N, T, osr, seed=N * 100 + T)
    nv = px.chan_vectors(N, T, D)
    x = px.int_samples(rng, N * T + nv * D + D // 2, True, lim=px.LIM)
    for name, steps in px.chan_patterns(N, T, D).items():
        calls = px.chan_run(N, taps, osr, x, steps)            # asserts the recovery
        assert calls[-1][3] == (0, 0, False)
        got = _chan_stream(calls)
        q = next(pos for (pos, _, _, (c, p, ca), _) in calls if p)   # the fill's completing call consumed nothing
        if N > 512:
            continue
        pushed = np.concatenate([x[:N * T], x[q:]])
        ref, ok = px.chan_textbook(N, D, taps, pushed, got.shape[1])
        assert ok.sum() >= nv // 2, (name, ok.sum())
        assert np.array_equal(got[:, ok], ref[:, ok]), name


def _synth_stream(calls):
    return np.concatenate([out[2] for (_, _, _, _, out) in calls])


@pytest.mark.parametrize("N,T,nofused", px.SYNTH_SHAPES)
def test_synth_oracle_exact(N, T, nofused):
    rng, taps = px.synth_case(N, T, seed=N * 100 + T)
    x, s = px.synth_inputs(rng, N, px.synth_vectors(N, T))
    streams = {}
    for name, steps in px.synth_patterns(N, T).items():
        calls = px.synth_run(N, taps, x, steps)                 # asserts the rounding
        streams[name] = _synth_stream(calls)
    ref, first = px.synth_textbook(N, taps, s)
    for name, z in streams.items():
        assert z.size == (s.shape[1] - T + 1) * N, name
        assert np.array_equal(z, streams["all"]), name
        assert np.array_equal(z[first:], ref), name


def _arb_stream(calls):
    return np.concatenate([out[0] for (_, _, _, cnt, out) in calls if cnt is not None])


@pytest.mark.parametrize("N,T,rate,periodic", px.PFBARB_SHAPES)
def test_pfbarb_oracle_patterns(N, T, rate, periodic):
    taps, x = px.pfbarb_case(N, T, rate, seed=N + T + int(rate * 1000))
    outs, _ = px.pfbarb_timing(rate, N, x.size - T)
    streams = {}
    for name, steps in px.pfbarb_patterns(rate, N, T, x.size - T).items():
        calls = px.pfbarb_run(rate, N, taps, x, steps)
        streams[name] = _arb_stream(calls)
    for name, y in streams.items():
        assert y.size == len(outs), name                        # the float32 timing loop counts like the oracle
        assert np.array_equal(y, streams["all"]), name          # call cuts and refused calls change nothing


@pytest.mark.parametrize("N,T,rate,periodic", px.PFBARB_HIGH_SHAPES)
def test_pfbarb_above_arm_count_patterns(N, T, rate, periodic):
    """Rates above the arm count (ArbRef, with the reference's saturating arm index): about `rate` outputs per sample for
    the whole stream -- a wrapping index stops the timing loop after the first Boundary output -- and every call pattern
    gives the same stream."""
    taps, x = px.pfbarb_case(N, T, rate, seed=N + T + int(rate * 1000))
    n = x.size - T
    outs, _ = px.pfbarb_timing(rate, N, n)
    if N > 1:                                  # (one arm: every step is a Boundary state, one output per sample)
        assert abs(len(outs) - n * np.float32(rate)) < 2 * rate
    else:
        assert len(outs) == n - 1                # (sample 0 only enters the Boundary state)
    streams = {name: _arb_stream(px.pfbarb_run(rate, N, taps, x, steps))
               for name, steps in px.pfbarb_patterns(rate, N, T, n).items()}
    for name, y in streams.items():
        assert y.size == len(outs), name
        assert np.array_equal(y, streams["all"]), name


@pytest.mark.parametrize("N,T,rate,periodic", px.PFBARB_SHAPES)
def test_arbref_equals_oracle(N, T, rate, periodic):
    """ArbRef (which stands in for the oracle above the arm count) is the oracle bit for bit wherever both apply."""
    taps, x = px.pfbarb_case(N, T, rate, seed=N + T + int(rate * 1000))
    steps = px.pfbarb_patterns(rate, N, T, x.size - T)["ragged"]
    want = px.pfbarb_run(rate, N, taps, x, steps)
    got = px.pfbarb_run(rate, N, taps, x, steps, ref=px.ArbRef)
    assert [c[:4] for c in got] == [c[:4] for c in want]
    assert np.array_equal(_arb_stream(got), _arb_stream(want))


@pytest.mark.parametrize("N,T,rate,periodic", px.PFBARB_SHAPES + px.PFBARB_HIGH_SHAPES)
def test_pfbarb_per_sample_bound(N, T, rate, periodic):
    """No sample produces more outputs than the descriptor tile of pfb_kernel is sized for."""
    outs, _ = px.pfbarb_timing(rate, N, 20000 if rate < 10 else 2000)
    per = np.bincount([o[0] for o in outs])
    assert per.max() <= px.pfbarb_per_sample_max(rate, N), (per.max(), px.pfbarb_per_sample_max(rate, N))


@pytest.mark.parametrize("rate", px.DYADIC_RATES)
@pytest.mark.parametrize("N,T", [(32, 5), (7, 3), (5, 1)])
def test_pfbarb_oracle_matches_textbook(rate, N, T):
    """At rates whose f32 delay is dyadic every mu is a multiple of 1/8 and every output an exact dyadic rational."""
    taps, x = px.pfbarb_case(N, T, 1.0, seed=3 * N + T)
    x = x[:T + 3000]
    y = _arb_stream(px.pfbarb_run(rate, N, taps, x, []))
    ref, ok = px.pfbarb_textbook(rate, N, taps, x)
    assert y.size == ref.size and ok.sum() > ref.size // 2
    assert np.array_equal(y[ok].astype(np.complex128), ref[ok])
    mus = np.array([float(m) for (_, _, m, _) in px.pfbarb_timing(rate, N, 3000)[0]])
    assert np.all(mus * 8 == np.rint(mus * 8))
