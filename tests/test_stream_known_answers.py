"""Replays tests/golden/reference_stream_known_answers.json: the reference's own known answers for Combine, Split,
firdes::hilbert and windows::hamming.  The tap design runs on the host (no GPU); the blocks run on the device through
VectorSource -> block -> VectorSink graphs wired exactly as the reference's tests wire them.

The fixture is transcribed by hand, with the file:line of each case: tests/combine.rs (three cases: equal lengths,
first input longer, second input longer), tests/split.rs, the Hilbert assertions of firdes/basic.rs:229-247 and the
MATLAB hamming() values of windows.rs:353-404 (tolerance 1e-5).  The blocks' u32 / i32 items become f32; every value
is exactly representable."""
import json
import os

import numpy as np
import pytest

import futuresdr_b200 as fb

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_stream_known_answers.json")))


def test_hamming_matches_matlab():
    c = GOLD["hamming"]
    w = fb.windows.hamming(c["len"], c["periodic"])
    assert w.dtype == np.float64 and w.size == c["len"]
    assert np.all(np.abs(w - np.asarray(c["window"])) < c["tolerance"]), c["cite"]


def test_hilbert_assertions():
    c = GOLD["hilbert"]
    taps = fb.firdes.hilbert(np.asarray(c["window"]))
    assert taps.dtype == np.float32 and taps.size == len(c["window"])
    assert all(taps[k] == 0.0 for k in c["zero_taps"]), c["cite"]
    assert all(abs(taps[a]) == abs(taps[b]) for a, b in c["equal_magnitude_pairs"]), c["cite"]
    assert all(taps[a] > taps[b] for a, b in c["strictly_greater"]), c["cite"]


def _gen_cos_literal(n, coeffs, periodic):
    """windows.rs:68-94 restated in Python floats (f64): alpha from f32, pi = f32::consts::PI widened."""
    npts = n + 1 if periodic else n
    alpha = float(np.float32(npts - 1) / np.float32(2.0))
    pi = float(np.float32(np.pi))
    out = []
    for i in range(npts):
        s = -0.0
        for k, ck in enumerate(coeffs):
            s += (-1.0) ** k * ck * np.cos(pi * float(k * i) / alpha)
        out.append(s)
    return np.asarray(out[:n])


def _hilbert_literal(window):
    """basic.rs:202-222 restated: the step_by(2) loop over 1..h and the gain recurrence, then x / gain as f32."""
    n = len(window)
    taps = [0.0] * n
    h = (n - 1) // 2
    gain = 0.0
    for i in range(1, h, 2):
        x = 1.0 / i
        taps[h + i] = x * window[h + i]
        taps[h - i] = -x * window[h - i]
        gain = taps[h + i] - gain
    gain = 2.0 * abs(gain)
    with np.errstate(invalid="ignore"):                       # n == 3: 0 / 0, NaN as in Rust
        return (np.asarray(taps) / np.float64(gain)).astype(np.float32)


@pytest.mark.parametrize("n,periodic", [(38, False), (38, True), (167, False), (64, True), (2, False), (1, True)])
def test_hamming_is_gen_cos_literally(n, periodic):
    assert np.array_equal(fb.windows.hamming(n, periodic), _gen_cos_literal(n, [0.54, 0.46], periodic))


@pytest.mark.parametrize("n", [3, 5, 11, 65, 167, 1001])
def test_hilbert_is_the_reference_loop(n):
    w = fb.windows.hamming(n)
    assert np.array_equal(fb.firdes.hilbert(w), _hilbert_literal(list(w)), equal_nan=True)


def test_hilbert_even_length_is_refused():
    from futuresdr_b200._lib import lib
    import ctypes as C
    w = np.ones(10)
    assert lib.b2s_firdes_hilbert(w.ctypes.data_as(C.POINTER(C.c_double)), 10, None, 0) == 0
    assert lib.b2s_firdes_hilbert(w.ctypes.data_as(C.POINTER(C.c_double)), 0, None, 0) == 0
    with pytest.raises(AssertionError, match="odd"):
        fb.firdes.hilbert(w)
    assert fb.windows.hamming(0).size == 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", GOLD["combine"], ids=[c["cite"].split()[-1] for c in GOLD["combine"]])
def test_combine_graph_reference_vectors(case):
    from futuresdr_b200.edges import Flowgraph, VectorSink, VectorSource
    fg = Flowgraph()
    src0 = VectorSource(np.asarray(case["in0"], np.float32))
    src1 = VectorSource(np.asarray(case["in1"], np.float32))
    combine = fb.Combine(fb.CombineOp.AddF32)
    snk = VectorSink(np.float32, case["sink_capacity"])
    fg.connect(src0, combine, "in0")                          # connect!(fg, src0 > in0.combine.output > snk)
    fg.connect(combine, snk)
    fg.connect(src1, combine, "in1")                          # connect!(fg, src1 > in1.combine)
    fg.run()
    v = snk.items()
    assert v.tolist() == [float(x) for x in case["output"]], case["cite"]


@pytest.mark.gpu
def test_split_graph_reference_vector():
    from futuresdr_b200.edges import Flowgraph, VectorSink, VectorSource
    case = GOLD["split"][0]
    x = (np.asarray(case["input_re"], np.float32) + 1j * np.asarray(case["input_im"], np.float32)).astype(np.complex64)
    fg = Flowgraph()
    src = VectorSource(x)
    split = fb.Split(fb.SplitOp.ReIm)
    snk0, snk1 = VectorSink(np.float32, 10), VectorSink(np.float32, 10)
    fg.connect(src, split)                                    # connect!(fg, src > input.split.output0 > snk0;
    fg.connect(split, "output0", snk0)                        #                split.output1 > snk1)
    fg.connect(split, "output1", snk1)
    fg.run()
    assert snk0.items().tolist() == [float(v) for v in case["output0"]], case["cite"]
    assert snk1.items().tolist() == [float(v) for v in case["output1"]], case["cite"]
