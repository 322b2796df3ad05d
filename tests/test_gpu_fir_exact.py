"""Every FIR, decimator and resampler path, bit for bit, on exactly representable inputs.

Samples and taps are small integers (tests/fir_exact.py), so every correct kernel -- whatever its summation order, FMA
use or bf16 split -- returns the exact integer sum, and any wrong tap, sample, phase, tile seam or device slot moves an
output by at least one unit.  That is what the tolerance tests (1e-5 * ||taps||_1 * max|x|) cannot see: a dropped
outer tap of a polyphase arm is far below their gate.  Values are compared, not bytes (-0.0 == 0.0: the tensor kernel
may differ in the sign of an exact zero, DESIGN.md 4.2); counts are compared exactly with the oracle's; every output
buffer is pre-filled with a non-integer sentinel that must survive outside [0, produced).

The shapes sit where the kernels change behaviour: the sliding-window kernel's tile (1024 outputs) and 16-byte vector
edges, its 160 KiB tile limit (fir_naive_kernel above it), the resampler's bank loop (L = 1..4 and >= 5) and the
general / one-thread-per-output resampler kernels, the tensor kernel's 16-wide K-steps, tiles, `lead` and detached
history, the overlap-save block length, and the host-slice pipeline's chunks and slots.  test_every_path_is_reached
checks with the profiler that the sweep reaches every one of these kernels.
"""
import os
import re
import sys

import numpy as np
import pytest

import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fir_exact as fx  # noqa: E402

pytestmark = pytest.mark.gpu

SENT = 4097.5                       # not an integer: no exact output equals it
KINDS = ["f32", "c32", "c32c"]      # samples x taps: f32 x f32, c32 x f32, c32 x c32


@pytest.fixture(scope="module")
def fb():
    import torch
    import futuresdr_b200 as fb
    assert torch.cuda.is_available()
    return fb


def _np_dtype(kind):
    return np.float32 if kind == "f32" else np.complex64


def _torch_dtype(kind):
    import torch
    return torch.float32 if kind == "f32" else torch.complex64


def _epc(kind):
    return 4 if kind == "f32" else 2          # items per 16 bytes


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _call(filt, kind, x_dev, n_in, cap, ioff=0, ooff=0):
    """filt.filter on x_dev[:n_in] placed `ioff` items past a 16-byte boundary (NaN in front), into an output slice
    `ooff` items past one, of capacity `cap`, sentinel everywhere.  Returns (counts, outputs, sentinel intact)."""
    import torch
    td = _torch_dtype(kind)
    buf = torch.full((ioff + n_in,), float("nan"), dtype=td, device="cuda")
    buf[ioff:] = x_dev[:n_in]
    out = torch.full((ooff + cap + 8,), SENT, dtype=td, device="cuda")
    c, p, st = filt.filter(buf[ioff:], out[ooff:ooff + cap])
    o = out.cpu().numpy()
    intact = bool(np.all(o[:ooff] == SENT) and np.all(o[ooff + p:] == SENT))
    return (c, p, int(st)), o[ooff:ooff + p], intact


def _exact(got, ref):
    return got.size == ref.size and np.array_equal(got.astype(ref.dtype), ref)


def _check_fir(filt, kind, x_dev, ref, N, D, n_out, cap=None, ioff=0, ooff=0, extra=0):
    n_in = n_out * D + N - 1 + extra
    cap = n_out if cap is None else cap
    counts, got, intact = _call(filt, kind, x_dev, n_in, cap, ioff, ooff)
    what = dict(kind=kind, N=N, D=D, n_out=n_out, cap=cap, ioff=ioff, ooff=ooff)
    assert counts == fx.fir_counts(n_in, N, D, cap), what
    assert intact, ("wrote outside [0, produced)", what)
    assert _exact(got, ref[:counts[1]]), (what, np.flatnonzero(got != ref[:got.size])[:8])


def _sweep_fir(fb, kind, N, D, algo, n_outs, seed):
    """One plan, one integer input long enough for max(n_outs); every n_out aligned with a full capacity, then again
    with input and output 1..EPC-1 items past a 16-byte boundary and capacities around n_out (some below it)."""
    rng = np.random.default_rng(seed)
    epc = _epc(kind)
    x = fx.int_samples(rng, max(n_outs) * D + N - 1 + D, kind != "f32")
    taps = fx.int_taps(rng, N, kind == "c32c")
    ref = fx.fir(taps, x, D)
    filt = fb.DecimatingFirFilter(D, taps, sample_dtype=_np_dtype(kind), algo=algo)
    xd = _dev(x)
    for j, n in enumerate(n_outs):
        _check_fir(filt, kind, xd, ref, N, D, n, extra=j % D)
        ioff, ooff = 1 + j % (epc - 1), 1 + (j // 2) % (epc - 1)
        cap = (n + 3, n - 1, n // 3, n)[j % 4]
        _check_fir(filt, kind, xd, ref, N, D, n, cap=max(cap, 0), ioff=ioff, ooff=ooff, extra=(D - 1 - j) % D)
    return filt


def _n_outs(kind):
    return [1, _epc(kind) - 1, 1023, 1024, 1025, 2047, 2049]


# ---- fir_direct_kernel, one bank (the FIR and the decimator) ----------------------------------------------------
DIRECT_NS = [1, 2, 7, 8, 9, 15, 16, 17, 63, 64, 65, 255, 256, 257, 1024, 4000]
DIRECT_DS = [1, 2, 3, 4, 5, 7, 8, 16, 19, 25, 38, 64]


@pytest.mark.parametrize("D", DIRECT_DS)
@pytest.mark.parametrize("kind", KINDS)
def test_direct_fir_exact(fb, kind, D):
    ns = {n for n in (1, D - 1, D, D + 1, 3 * D + 1) if n >= 1}
    ns |= set(DIRECT_NS if D <= 4 else (8, 17, 64, 257))
    for N in sorted(ns):
        _sweep_fir(fb, kind, N, D, fb.ALGO_DIRECT, _n_outs(kind), seed=1000 * N + D)


# ---- fir_naive_kernel: on both sides of the 160 KiB tile limit ----------------------------------------------------
@pytest.mark.parametrize("kind,D,N", [("c32", 19, 9), ("c32", 20, 9), ("c32", 20, 64), ("c32c", 19, 9), ("c32c", 20, 33),
                                      ("f32", 38, 17), ("f32", 39, 17), ("f32", 127, 5), ("f32", 128, 256),
                                      ("f32", 1000, 3), ("c32", 1, 12960), ("c32", 1, 12961), ("c32", 1, 13000),
                                      ("c32c", 1, 13000), ("f32", 1, 20000)])
def test_direct_fir_tile_limit_exact(fb, kind, D, N):
    _sweep_fir(fb, kind, N, D, fb.ALGO_DIRECT, _n_outs(kind), seed=7 * N + D)


# ---- many waves, and one long call per kind ------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_direct_fir_long_exact(fb, kind):
    rng = np.random.default_rng(11)
    for N, D, n_out in ((63, 1, 200 * 1024 - 1), (17, 3, 200 * 1024 + 1), (64, 1, 16 * 1024 * 1024 - 3)):
        x = fx.int_samples(rng, n_out * D + N - 1, kind != "f32")
        taps = fx.int_taps(rng, N, kind == "c32c")
        filt = fb.DecimatingFirFilter(D, taps, sample_dtype=_np_dtype(kind), algo=fb.ALGO_DIRECT)
        _check_fir(filt, kind, _dev(x), fx.fir(taps, x, D), N, D, n_out)


# ---- fir_tc_kernel ------------------------------------------------------------------------------------------------
TC_NS = [16, 17, 23, 24, 31, 32, 48, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257]
TC_DS = [1, 2, 4, 8, 16, 32, 64, 128]


def _tile(kind):
    return 8192 if kind == "c32" else 16384       # full-rate items per tensor tile


_tc_input = {}


def _tc_x(kind):
    """One integer input per sample type, long enough for more tiles than 2 x SMs (shared by every N)."""
    import torch
    if kind not in _tc_input:
        tiles = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 5
        x = fx.int_samples(np.random.default_rng(5), tiles * _tile(kind) + 512, kind != "f32")
        _tc_input[kind] = (x, _dev(x), tiles)
    return _tc_input[kind]


@pytest.mark.parametrize("N", TC_NS)
@pytest.mark.parametrize("kind", ["f32", "c32"])
def test_tensor_fir_exact(fb, kind, N):
    """Every D | 128 and every `lead` (slice 0..EPC-1 items past a 16-byte boundary; at N + lead > 257 the call falls
    back to the direct kernel, which must be exact too), n_out around one and three tiles, small capacities (the
    epilogue's room mask), and one call over more tiles than 2 x SMs."""
    x, xd, tiles = _tc_x(kind)
    taps = fx.int_taps(np.random.default_rng(N), N)
    y = fx.conv_valid(x, taps)                       # full rate: the decimated references are slices of it
    for D in TC_DS:
        filt = fb.DecimatingFirFilter(D, taps, sample_dtype=_np_dtype(kind), algo=fb.ALGO_TENSOR)
        assert filt.algo == fb.ALGO_TENSOR
        ref = y[D - 1::D]
        per_tile = _tile(kind) // D
        for lead in range(_epc(kind)):
            for n in (per_tile - 1, per_tile, per_tile + 1, 3 * per_tile + 5):
                _check_fir(filt, kind, xd, ref, N, D, n, ioff=lead, extra=(lead * 5) % D)
            if D > 1:
                for cap in (1, 5, per_tile // 2 + 3):
                    _check_fir(filt, kind, xd, ref, N, D, 3 * per_tile, cap=cap, ioff=lead)
        if D in (1, 4):
            n_many = (tiles - 1) * _tile(kind) // D + 3
            _check_fir(filt, kind, xd, ref, N, D, n_many, ioff=D // 4)


def _exec_hist(filt, hist, inp, out):
    import ctypes as C
    from futuresdr_b200._lib import lib, check
    c, p, st = C.c_size_t(0), C.c_size_t(0), C.c_int32(0)
    check(lib.b2s_fir_exec_hist(filt._h, C.c_void_p(hist.data_ptr()), hist.numel(), C.c_void_p(inp.data_ptr()),
                                inp.numel(), C.c_void_p(out.data_ptr()), out.numel(), None, C.byref(c), C.byref(p),
                                C.byref(st)), filt.ctx.handle)
    return c.value, p.value, st.value


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("N,D", [(24, 1), (64, 1), (129, 2), (255, 1), (256, 1), (257, 1), (52, 4), (100, 16), (200, 128)])
@pytest.mark.parametrize("kind", ["f32", "c32"])
def test_tensor_exec_hist_exact(fb, kind, N, D, fused):
    """b2s_fir_exec_hist with a detached history of H = ceil((N-1)/D)*D items (fused: the kernel fetches it, lead +
    n_hist <= 1024) or of H + 1024 items (copied in front of the slice first).  Everything around the history and the
    slice that is not part of the logical input is NaN."""
    import torch
    td, q = _torch_dtype(kind), _epc(kind)
    H = -(-(N - 1) // D) * D
    n_hist = H if fused else H + 1024
    lead = (-n_hist) % q
    n_in = 3 * _tile(kind) + 77
    rng = np.random.default_rng(N + 1000 * D)
    x = fx.int_samples(rng, n_hist + n_in, kind == "c32")
    taps = fx.int_taps(rng, N)
    filt = fb.DecimatingFirFilter(D, taps, sample_dtype=_np_dtype(kind), algo=fb.ALGO_TENSOR)
    hbuf = torch.full((lead + n_hist + 16,), float("nan"), dtype=td, device="cuda")
    hbuf[lead:lead + n_hist] = _dev(x[:n_hist])
    pad = -(-n_hist // 64) * 64
    ibuf = torch.full((pad + n_in,), float("nan"), dtype=td, device="cuda")
    ibuf[pad:] = _dev(x[n_hist:])
    ref = fx.fir(taps, x, D)
    for cap in (ref.size, ref.size // 2 + 1):
        out = torch.full((cap + 8,), SENT, dtype=td, device="cuda")
        c, p, st = _exec_hist(filt, hbuf[lead:lead + n_hist], ibuf[pad:], out[:cap])
        o = out.cpu().numpy()
        assert (c, p, st) == fx.fir_counts(n_hist + n_in, N, D, cap)
        assert np.all(o[p:] == SENT)
        assert _exact(o[:p], ref[:p])


# ---- the rational resampler ------------------------------------------------------------------------------------------
# (L, M) -> kernel with the default design (FirBuilder::resampling: kaiser_multirate(L, M, 12, 1e-4)):
#   sliding window (fir_direct_kernel): 1/10 (LT 1), 2/3 and 2/1 (LT 2), 3/2 (LT 3), 4/3 and 4/5 (LT 4), 5/1 and 8/3
#   (LT 0, a run-time loop over the banks); f32 also 1/11, 1/19 and 6/7;
#   resamp_kernel, taps in shared memory: c32 1/11, 1/19 and 6/7, 48/125, 160/147 and 147/160;
#   resamp_kernel, taps in global memory: c32 1/23;
#   resamp_naive_kernel (the span does not fit one tile): c32 1/25 ... 10/300, f32 1/51 and 1/100.
# test_every_path_is_reached confirms the mapping.
RS_RATIOS = [(1, 10), (2, 3), (2, 1), (3, 2), (4, 3), (4, 5), (5, 1), (8, 3), (1, 11), (1, 19), (6, 7), (48, 125),
             (160, 147), (147, 160), (1, 23), (1, 25), (1, 26), (1, 32), (1, 48), (1, 100), (2, 51), (3, 80), (4, 125),
             (10, 300), (1, 51)]


def _default_T(L, M):
    return orc.kaiser_multirate(L, M, 12, 1e-4).size // L


@pytest.mark.parametrize("T", [1, 2, 5, "default"])
@pytest.mark.parametrize("L,M", RS_RATIOS)
@pytest.mark.parametrize("kind", ["f32", "c32"])
def test_resampler_exact(fb, kind, L, M, T):
    T = _default_T(L, M) if T == "default" else T
    rng = np.random.default_rng(L * 1000 + M + 7 * T)
    n_target = 3 * 1024 * L + 5 if L <= 8 else 8000          # several tiles of either kernel
    n_in = (n_target * M) // L + T + M
    x = fx.int_samples(rng, n_in, kind == "c32")
    taps = fx.int_taps(rng, L * T)
    filt = fb.PolyphaseResamplingFir(L, M, taps, sample_dtype=_np_dtype(kind))
    xd = _dev(x)
    _, p_all, _ = fx.resamp_counts(n_in, L, M, T, 10 ** 9)
    ref = fx.resamp(taps, L, M, x, p_all)
    epc = _epc(kind)
    # whole input; then capacities that are not multiples of L on unaligned slices (vec_ok = 0)
    for cap, ioff, ooff in ((p_all + L + 3, 0, 0), (p_all - 1 - L // 2, 1, 1), (L + 1, epc - 1, 0),
                            (2 * L - 1, 0, epc - 1), (p_all // 2 + 1, 1, 0)):
        counts, got, intact = _call(filt, kind, xd, n_in, max(cap, 0), ioff, ooff)
        assert counts == fx.resamp_counts(n_in, L, M, T, max(cap, 0)), (cap, ioff, ooff)
        assert intact and _exact(got, ref[:counts[1]]), (cap, ioff, ooff)
    # a ragged call sequence, stitched: each call sees the unconsumed rest plus the next `step` items
    outs, pos, end = [], 0, 0
    for step in (3, 1, T, 4097, n_in):
        end = min(end + step, n_in)
        (c, p, st), got, intact = _call(filt, kind, xd[pos:], end - pos, p_all + L)
        assert (c, p, st) == fx.resamp_counts(end - pos, L, M, T, p_all + L) and intact
        outs.append(got)
        pos += c
    got = np.concatenate(outs)
    assert got.size == p_all and _exact(got, ref)


# ---- overlap-save (fir_fft.cu) ------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [64, 258, 1024, 2049])
@pytest.mark.parametrize("ctaps", [False, True])
def test_overlap_save_fir_near_exact(fb, ctaps, N):
    """Not exact (f32 FFTs), but any index error moves an output by at least 1: gate 0.25, with samples and taps in
    [-2, 2] so that the transform error stays far below it (the largest error is printed)."""
    V = 4096 - (N - 1)
    n_outs = [1, V - 1, V, V + 1, 2 * V, 2 * V + 1, 3 * V - 1, 5 * V + 7]
    rng = np.random.default_rng(N + ctaps)
    x = fx.int_samples(rng, max(n_outs) + N - 1 + 3, True, lim=2)
    taps = fx.int_taps(rng, N, ctaps, lim=2)
    filt = fb.FirFilter(taps, algo=fb.ALGO_FFT)
    assert filt.algo == fb.ALGO_FFT
    ref = fx.fir(taps, x)
    xd = _dev(x)
    worst = 0.0
    for j, n in enumerate(n_outs):
        cap = n if j % 3 else n + 5
        n_in = n + N - 1 + j % 3
        counts, got, intact = _call(filt, "c32", xd, n_in, cap)
        assert counts == fx.fir_counts(n_in, N, 1, cap) and intact
        err = float(np.max(np.abs(got.astype(np.complex128) - ref[:got.size]))) if got.size else 0.0
        worst = max(worst, err)
    print(f"overlap-save N={N} complex_taps={ctaps}: largest |y - y_exact| = {worst:.3g}")
    assert worst <= 0.25


# ---- host slices (b2s_fir_filter_host): several chunks per call, every slot reused -----------------------------------
_host_cases = {}


def _host_case(kind, D, N):
    """~26 Mi c32 / ~52 Mi f32 input items: at the default 32 MiB per chunk that is 6-7 chunks over 4 device slots."""
    key = (kind, D, N)
    if key not in _host_cases:
        _host_cases.clear()
        rng = np.random.default_rng(D * 100 + N)
        n_out = (26 << 20) // D if kind == "c32" else 52 << 20
        x = fx.int_samples(rng, n_out * D + N - 1, kind == "c32")
        taps = fx.int_taps(rng, N)
        _host_cases[key] = (x, taps, n_out, fx.fir(taps, x, D))
    return _host_cases[key]


@pytest.mark.parametrize("algo", ["direct", "tensor", "auto"])
@pytest.mark.parametrize("kind,D", [("c32", 1), ("c32", 4), ("f32", 1)])
def test_host_slices_exact(fb, kind, D, algo):
    N = 255
    x, taps, n_out, ref = _host_case(kind, D, N)
    filt = fb.DecimatingFirFilter(D, taps, sample_dtype=_np_dtype(kind),
                                  algo={"direct": fb.ALGO_DIRECT, "tensor": fb.ALGO_TENSOR, "auto": fb.ALGO_AUTO}[algo])
    out = np.full(n_out + 100, SENT, _np_dtype(kind))
    c, p, st = filt.filter(x, out)
    assert (c, p, int(st)) == fx.fir_counts(x.size, N, D, out.size) and p == n_out
    assert np.all(out[p:] == SENT)
    bad = np.flatnonzero(out[:p] != ref)
    assert bad.size == 0, ("first wrong outputs", bad[:8], "chunk of 32 MiB input", bad[:8] * D * x.itemsize >> 25)


# ---- the sweep reaches every kernel ---------------------------------------------------------------------------------
def test_every_path_is_reached(fb):
    """Runs a representative subset of the shapes above under the profiler and asserts which kernels ran: if a change
    to the selection rules moves a path off its kernel, the sweep no longer covers that kernel and this fails."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    rng = np.random.default_rng(3)

    def fir(kind, N, D, algo, n_out=3000):
        x = fx.int_samples(rng, n_out * D + N - 1, kind != "f32")
        taps = fx.int_taps(rng, N, kind == "c32c")
        f = fb.DecimatingFirFilter(D, taps, sample_dtype=_np_dtype(kind), algo=algo)
        _check_fir(f, kind, _dev(x), fx.fir(taps, x, D), N, D, n_out)

    def rs(kind, L, M):
        T = _default_T(L, M)
        n_in = 3000 * M // L + T + M
        x = fx.int_samples(rng, n_in, kind == "c32")
        taps = fx.int_taps(rng, L * T)
        f = fb.PolyphaseResamplingFir(L, M, taps, sample_dtype=_np_dtype(kind))
        counts, got, intact = _call(f, kind, _dev(x), n_in, 10 ** 6)
        assert intact and _exact(got, fx.resamp(taps, L, M, x, counts[1]))

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for kind in ("f32", "c32"):
            fir(kind, 9, 1, fb.ALGO_DIRECT)
            fir(kind, 64, 4, fb.ALGO_TENSOR)
            for L, M in ((1, 10), (2, 3), (3, 2), (4, 5), (8, 3), (48, 125), (1, 100)):
                rs(kind, L, M)
        fir("c32c", 9, 20, fb.ALGO_DIRECT)
        fir("f32", 9, 39, fb.ALGO_DIRECT)
        rs("c32", 1, 23)
        x, taps = fx.int_samples(rng, 9000, True, lim=2), fx.int_taps(rng, 1024, lim=2)
        counts, got, intact = _call(fb.FirFilter(taps, algo=fb.ALGO_FFT), "c32", _dev(x), x.size, x.size)
        assert intact and np.max(np.abs(got - fx.fir(taps, x))) <= 0.25
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    found = set()
    for n in names:
        m = re.search(r"fir_direct_kernel<(float2?), (float2?), (\d)>", n)
        if m:
            found.add(("direct", m.group(1), int(m.group(3))))
        m = re.search(r"resamp_kernel<(float2?), (true|false)>", n)
        if m:
            found.add(("resamp", m.group(1), m.group(2)))
        for k in ("fir_naive_kernel", "resamp_naive_kernel", "fir_fft_kernel"):
            if re.search(k + "<", n):
                found.add((k,))
        m = re.search(r"fir_tc_kernel<(true|false)>", n)
        if m:
            found.add(("tc", m.group(1)))
    want = {("direct", s, lt) for s in ("float", "float2") for lt in range(5)}
    want |= {("resamp", "float", "true"), ("resamp", "float2", "true"), ("resamp", "float2", "false")}
    want |= {("fir_naive_kernel",), ("resamp_naive_kernel",), ("fir_fft_kernel",), ("tc", "true"), ("tc", "false")}
    assert want <= found, (sorted(want - found), sorted(n for n in names if "kernel" in n))
