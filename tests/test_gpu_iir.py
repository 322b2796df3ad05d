"""IirFilter / Iir on the GPU (csrc/iir.cu) against the CPU oracle (tests/iir_oracle.py, iir.rs:78-178).

DIRECT (the sequential kernel) must equal the oracle bit for bit; SCAN (the chained scan) is gated against the exact
f64 recurrence and the f32 reference:
  (a) max|y - y_exact| <= max(1e-5 G max|x|, 2 max|y_ref - y_exact|)
  (b) max|y - y_ref|   <= 1e-5 G max|x| + max|y_ref - y_exact|
with G = ||h||_1 + sum_j ||g_j||_1 (impulse response plus the zero-input responses to unit initial memory)."""
import json
import os
import sys

import numpy as np
import pytest
import torch
from scipy import signal

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import iir_oracle as orc  # noqa: E402  (tests/iir_oracle.py)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_iir_known_answers.json")))["cases"]
N_BIG = 64 << 20


def fb():
    import futuresdr_b200 as m
    return m


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def run_calls(f, xd, calls, dtype=torch.float32):
    """Drive a StatefulFilter like a block does: each call sees the unconsumed input from `pos`, `calls` are
    (input length, output capacity) pairs.  Returns the concatenated output and the (c, p, status) triples."""
    pos, outs, trip = 0, [], []
    for n, cap in calls:
        o = torch.empty(max(cap, 1), dtype=dtype, device="cuda")
        c, p, st = f.filter(xd[pos: pos + n], o[:cap])
        trip.append((c, p, int(st)))
        outs.append(o[:p])
        pos += c
    return torch.cat(outs), trip


def gain_bound(a, b):
    """G = ||h||_1 + sum_j ||g_j||_1 in f64 (a in the reference's sign convention)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    aa = np.concatenate([[1.0], -a])
    r = float(np.max(np.abs(np.roots(aa)))) if a.size else 0.0
    L = int(min(1 << 23, 64 + (np.log(1e-14) / np.log(r) if 0 < r < 1 else 64)))
    imp = np.zeros(L + b.size)
    imp[0] = 1.0
    G = float(np.sum(np.abs(signal.lfilter(b, aa, imp))))
    for j in range(a.size):
        e = np.zeros(a.size)
        e[j] = 1.0
        zi = signal.lfiltic([1.0], aa, e)
        G += float(np.sum(np.abs(signal.lfilter([1.0], aa, np.zeros(L), zi=zi)[0])))
    return G


def check_gate(ys, a, b, x, G=None):
    """Gates (a) and (b) for one output stream or a list of them (all of the same input)."""
    y_ref = orc.iir(a, b, x).astype(np.float64)
    y_ex = orc.iir_exact(a, b, x)
    G = gain_bound(a, b) if G is None else G
    tol = 1e-5 * G * float(np.max(np.abs(x)))
    ref_err = float(np.max(np.abs(y_ref - y_ex)))
    for y in ys if isinstance(ys, list) else [ys]:
        y = np.asarray(y, np.float64)
        assert y.shape == y_ref.shape == y_ex.shape
        err_ex = float(np.max(np.abs(y - y_ex)))
        err_ref = float(np.max(np.abs(y - y_ref)))
        assert err_ex <= max(tol, 2 * ref_err), (err_ex, tol, ref_err)          # (a)
        assert err_ref <= tol + ref_err, (err_ref, tol, ref_err)                 # (b)
    return err_ex, err_ref, tol, ref_err


def one_pole(r):
    return [r], [1.0]


def butter(order, wn=0.1):
    bb, aa = signal.butter(order, wn)
    return list(-aa[1:]), list(bb)                 # reference convention: y += a[j] * y[k-1-j]


def random_poles(seed, n_b):
    rng = np.random.default_rng(seed)
    mag = rng.uniform(0.3, 0.95, 4)
    ang = rng.uniform(0.05, np.pi - 0.05, 4)
    poles = np.concatenate([mag * np.exp(1j * ang), mag * np.exp(-1j * ang)])
    aa = np.real(np.poly(poles))
    return list(-aa[1:]), list(rng.uniform(-1, 1, n_b))


FILTERS = {f"pole{r}": one_pole(r) for r in (0.5, 0.9, 0.99, 0.999, 0.9999)}
FILTERS["dc_blocker"] = ([0.995], [1.0, -1.0])
FILTERS.update({f"butter{o}": butter(o) for o in (2, 4, 6)})
FILTERS.update({f"rand8_nb{nb}": random_poles(100 + nb, nb) for nb in (1, 9, 64)})


@pytest.fixture(scope="module")
def noise():
    return np.random.default_rng(0x11).standard_normal(N_BIG).astype(np.float32)


def inputs(noise, kind):
    if kind == "noise":
        return noise
    if kind == "dc":
        return np.ones(N_BIG, np.float32)
    if kind == "nyquist":
        return np.where(np.arange(N_BIG) % 2 == 0, 1.0, -1.0).astype(np.float32)
    if kind == "tiny":
        return (noise * np.float32(1e-20)).astype(np.float32)
    return (noise * np.float32(1e15)).astype(np.float32)


# ---- reference vectors ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
@pytest.mark.parametrize("algo", ["auto", "direct", "scan"])
def test_reference_vectors_through_the_abi(case, algo):
    m = fb()
    f = m.IirFilter(case["a"], case["b"], np.float32)
    if algo == "direct":
        f.set_algo(m.ALGO_DIRECT)
    elif algo == "scan":
        if not case["a"] or case["name"] == "doc_example":          # n_a == 0 / unstable: not admitted
            with pytest.raises(m.B200SdrError) as e:
                f.set_algo(m.ALGO_SCAN)
            assert e.value.code == m._lib.EUNSUPPORTED
            return
        f.set_algo(m.ALGO_SCAN)
    assert f.length() == len(case["b"])
    if case["mode"] == "feeder":
        buf, outs = [], []
        for v in case["input"]:
            buf.append(v)
            o = torch.zeros(1, device="cuda")
            c, p, _ = f.filter(torch.tensor(buf, dtype=torch.float32, device="cuda"), o)
            assert c == p
            del buf[:c]
            outs.append(float(o[0]) if p else None)
        assert outs == case["expected"]
    else:
        o = torch.zeros(case["out_cap"], device="cuda")
        c, p, _ = f.filter(dev(np.float32(case["input"])), o)
        assert (c, p) == (1, 1) and o.cpu().tolist() == case["expected"]


# ---- counts / status -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("algo", ["auto", "direct"])
@pytest.mark.parametrize("n_a,n_b", [(0, 1), (0, 4), (1, 1), (3, 1), (3, 5), (8, 64)])
def test_counts_and_values_on_ragged_calls(algo, n_a, n_b):
    m = fb()
    rng = np.random.default_rng(7 * n_a + n_b)
    a = (rng.uniform(-1, 1, n_a) * 0.9 / max(n_a, 1)).astype(np.float32)
    b = rng.uniform(-1, 1, n_b).astype(np.float32)
    x = rng.standard_normal(200_000).astype(np.float32)
    f = m.IirFilter(a, b, np.float32, algo=m.ALGO_DIRECT if algo == "direct" else m.ALGO_AUTO)
    o = orc.Iir(a, b)
    sizes = [0, 1, max(n_a - 1, 0), n_a, max(n_b - 1, 0), 2, 0, 5000, 70_000, 100_000]
    calls = [(s, int(rng.choice([0, 1, s, s + 7, max(s // 3, 1)]))) for s in sizes]
    yd, trip = run_calls(f, dev(x), calls)
    pos, want, ys = 0, [], []
    for n, cap in calls:
        c, p, st, y = o.filter(x[pos: pos + n], cap)
        want.append((c, p, st))
        ys.append(y)
        pos += c
    assert trip == want
    y_ref = np.concatenate(ys)
    if f.algo == m.ALGO_DIRECT and (n_a or algo == "direct"):
        np.testing.assert_array_equal(yd.cpu().numpy().view(np.uint32), y_ref.view(np.uint32))
    else:
        assert np.max(np.abs(yd.cpu().numpy() - y_ref)) <= 1e-5 * gain_bound(a, b) * np.max(np.abs(x))


def test_fill_split_across_calls_and_empty_slices():
    m = fb()
    a, b = [0.25, -0.125, 0.0625], [1.0, 0.5]
    f, o = m.IirFilter(a, b, np.float32), orc.Iir(a, b)
    x = np.float32([3, -1, 4, 1, -5, 9, 2, -6, 5, 3])
    xd = dev(x)
    pos = 0
    for n, cap in [(0, 0), (0, 4), (1, 4), (2, 0), (2, 4), (3, 0), (3, 1), (10, 10), (10, 10)]:
        out = torch.zeros(max(cap, 1), device="cuda")
        c, p, st = f.filter(xd[pos: pos + n], out[:cap])
        c2, p2, st2, y = o.filter(x[pos: pos + n], cap)
        assert (c, p, int(st)) == (c2, p2, st2), (n, cap)
        assert out[:p].cpu().numpy().tobytes() == y.tobytes()
        pos += c


# ---- DIRECT: bit-identical -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", ["biquad", "n_a7_n_b1", "fir3"])
def test_direct_bit_identical_with_denormals_and_nonfinite(dtype, shape):
    m = fb()
    rng = np.random.default_rng(3)
    if shape == "biquad":
        a, b = butter(2)
    elif shape == "n_a7_n_b1":
        a, b = list(rng.uniform(-0.12, 0.12, 7)), [1.0]
    else:
        a, b = [], [0.25, 0.5, 0.25]
    a, b = np.asarray(a, dtype), np.asarray(b, dtype)
    n = 4 << 20
    x = rng.standard_normal(n).astype(dtype)
    tiny = np.finfo(dtype).tiny
    x[1000:9000] = 0                                            # the state decays below the normal range ...
    x[9000:9100] = tiny * rng.uniform(-0.5, 0.5, 100)           # ... and denormal samples enter it
    x[n - 3000] = np.inf
    x[n - 2000] = np.nan
    x[n - 1000] = -np.inf
    f = m.IirFilter(a, b, dtype, algo=m.ALGO_DIRECT)
    assert f.algo == m.ALGO_DIRECT
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    y = torch.empty(n, dtype=tdt, device="cuda")
    c, p, _ = f.filter(dev(x), y)
    f.ctx.sync()
    y = y[:p].cpu().numpy()
    y_ref = orc.iir(a, b, x, dtype)
    assert p == y_ref.size == n - b.size + 1
    nan = np.isnan(y_ref)
    assert np.array_equal(np.isnan(y), nan)                     # NaN payloads may differ between CPU and GPU
    assert np.array_equal(y[~nan].view(np.uint8), y_ref[~nan].view(np.uint8))
    assert np.any((y != 0) & (np.abs(y) < tiny))                # denormal outputs were compared


# ---- SCAN: gated numerics --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(FILTERS))
def test_scan_gates(name, noise):
    m = fb()
    a, b = FILTERS[name]
    a32, b32 = np.float32(a), np.float32(b)
    f = m.IirFilter(a32, b32, np.float32)
    assert f.algo == m.ALGO_SCAN, name
    G = gain_bound(a32, b32)
    kinds = ["noise", "dc", "nyquist", "tiny", "huge"] if not name.startswith("rand") else ["noise", "dc"]
    for kind in kinds:
        x = inputs(noise, kind)
        f = m.IirFilter(a32, b32, np.float32, algo=m.ALGO_SCAN)
        y = torch.empty(N_BIG, device="cuda")
        c, p, _ = f.filter(dev(x), y)
        f.ctx.sync()
        assert p == N_BIG - b32.size + 1
        errs = check_gate(y[:p].cpu().numpy(), a32, b32, x, G)
        print(name, kind, "err_exact %.3e err_ref %.3e tol %.3e ref_err %.3e" % errs)


@pytest.mark.parametrize("bad", [np.nan, np.inf])
@pytest.mark.parametrize("name", ["pole0.99", "butter4", "rand8_nb9"])
def test_scan_nonfinite_set_equals_reference(name, bad):
    m = fb()
    a, b = np.float32(FILTERS[name][0]), np.float32(FILTERS[name][1])
    n = 1 << 22
    x = np.random.default_rng(9).standard_normal(n).astype(np.float32)
    x[3 * n // 4 + 123] = bad
    f = m.IirFilter(a, b, np.float32, algo=m.ALGO_SCAN)
    y = torch.empty(n, device="cuda")
    c, p, _ = f.filter(dev(x), y)
    f.ctx.sync()
    y_ref = orc.iir(a, b, x)
    assert np.array_equal(np.isfinite(y[:p].cpu().numpy()), np.isfinite(y_ref))
    assert not np.isfinite(y_ref[3 * n // 4 + 123 - b.size + 1])


@pytest.mark.parametrize("name", ["pole0.999", "butter6", "rand8_nb64"])
def test_scan_one_call_equals_ragged_calls(name, noise):
    m = fb()
    a, b = np.float32(FILTERS[name][0]), np.float32(FILTERS[name][1])
    x = noise
    xd = dev(x)
    f1 = m.IirFilter(a, b, np.float32, algo=m.ALGO_SCAN)
    y1 = torch.empty(N_BIG, device="cuda")
    _, p1, _ = f1.filter(xd, y1)
    rng = np.random.default_rng(11)
    calls, total = [(0, 0), (1, 1), (len(a) - 1, 5), (len(a), 0)], 0
    while total < N_BIG:
        s = int(rng.choice([1, 7, 4095, 4096, 4097, 100_003, 3_000_000, 9_000_001]))
        calls.append((s, s))
        total += s
    calls.append((N_BIG, N_BIG))
    f2 = m.IirFilter(a, b, np.float32, algo=m.ALGO_SCAN)
    y2, _ = run_calls(f2, xd, calls)
    f2.ctx.sync()
    assert y2.numel() == p1
    G = gain_bound(a, b)
    check_gate([y1[:p1].cpu().numpy(), y2.cpu().numpy()], a, b, x, G)


def test_scan_refused_and_auto_resolves_to_direct():
    m = fb()
    plans = {
        "n_a9": (np.float32(np.full(9, 0.05)), np.float32([1.0]), np.float32),
        "unstable": (np.float32([1.5, -0.2]), np.float32([1.0]), np.float32),
        "r1": (np.float32([1.0]), np.float32([1.0]), np.float32),
        "f64": (np.float64([0.5]), np.float64([1.0]), np.float64),
        "n_b65": (np.float32([0.5]), np.float32(np.ones(65)), np.float32),
    }
    for name, (a, b, dt) in plans.items():
        f = m.IirFilter(a, b, dt)
        assert f.algo == m.ALGO_DIRECT, name
        with pytest.raises(m.B200SdrError) as e:
            f.set_algo(m.ALGO_SCAN)
        assert e.value.code == m._lib.EUNSUPPORTED, name
    f = m.IirFilter([0.5], [1.0], np.float32)
    assert f.algo == m.ALGO_SCAN
    with pytest.raises(m.B200SdrError):
        f.set_algo(m.ALGO_TENSOR)
    fir = m.FirFilter([1.0, 2.0, 3.0], sample_dtype=np.float32)
    with pytest.raises(m.B200SdrError) as e:
        fir.set_algo(m.ALGO_SCAN)
    assert e.value.code == m._lib.EUNSUPPORTED
    with pytest.raises(m.B200SdrError) as e:
        m.IirFilter([0.5], [], np.float32)
    assert e.value.code == m._lib.EINVAL


# ---- block -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_iir_block_under_mocker_equals_oracle(dtype):
    from futuresdr_b200 import blocks as B
    a, b = butter(2)
    x = np.random.default_rng(4).standard_normal(100_000).astype(dtype)
    blk = B.IirBuilder.same_type(a, b, dtype)
    assert blk.input.min_items == len(b)
    mk = B.Mocker(blk)
    mk.input(x)
    mk.init_output(x.size)
    mk.run()
    y = mk.output().cpu().numpy()
    y_ref = orc.iir(np.asarray(a, dtype), np.asarray(b, dtype), x, dtype)
    if dtype == np.float64:
        assert np.array_equal(y, y_ref)
    else:
        check_gate(y, np.float32(a), np.float32(b), x)
