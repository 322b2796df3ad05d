"""Exact references for the three polyphase filter banks on integer data (test infrastructure).

Samples and taps are small integers (fir_exact.int_samples / int_taps), so every arm dot product is an integer below
2^24 and every correct kernel returns it exactly, whatever its summation order or FMA use.  Each block is then checked
exactly:

* PfbArbResampler: bit for bit against the oracle.  The arm dots are exact in both, and the blend
  (1-mu)*y0 + mu*y1 is the same sequence of separately rounded IEEE operations on both sides.
* PfbChannelizer: in the arm domain.  An output vector is the un-normalised inverse DFT of the N integer arm outputs;
  chan_arms() recovers them as FFT_f64(y)/N.  The map is unitary up to sqrt(N), so a wrong arm value moves some
  channel by at least 1, while the f32 transform error divided by sqrt(N) stays far below 0.25.
* PfbSynthesizer: integer outputs by construction.  synth_inputs() feeds x = FFT_f64(s)/N for integer "spun"
  vectors s, so the inverse FFT inside the block returns s to within ~1e-6 and every output is an integer to within a
  small fraction; a wrong tap or spun sample moves an output by a whole unit.

The drivers run the CPU oracle through a sequence of work() calls and return, per call, the counts and the expected
values; the device tests make the same calls.  The textbook functions restate each block's steady state in float64
and are used only to cross-check the oracle (itself a restatement) on the CPU.

The shape lists sit where the device code changes behaviour; the GPU tests and the CPU cross-check share them.
"""
from __future__ import annotations

import os
import sys

import numpy as np

import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fir_exact import int_samples, int_taps  # noqa: E402,F401

LIM = 4                                  # samples and taps in [-4, 4]
RECOVER_TOL = 1e-3                       # the oracle's own distance from the integers it stands for


# ---- geometry of the fused kernels (pfb_common.cuh, fft_common.cuh) -------------------------------------------------
def fused_tpad(N, T):
    """pfb_fused_tpad: the padded tap count of the fused banks, 0 where they do not apply."""
    if N < 4 or N > 256 or N & (N - 1) or T > 32:
        return 0
    return 8 if T <= 8 else (16 if T <= 16 else 32)


def fused_ob(N):
    """Output vectors per fused tile: fft_geom(log2 N, 256).fpb."""
    return 256 // max(1, min(N // 16, 256))


def synth_lead(N, T):
    """Vectors at the start of a steady synthesizer call that stay on the generic path (synth_fused_lead)."""
    ob, tpad = fused_ob(N), fused_tpad(N, T)
    return -(-(tpad - 1) // ob) * ob if tpad else 0


# ---- shapes ---------------------------------------------------------------------------------------------------------
TS = [1, 2, 3, 4, 5, 8, 9, 16, 17, 31, 32]

# (N, T, oversample_rate, no_fused)
CHAN_SHAPES = ([(N, T, 1.0, False) for N in (4, 8, 64, 256) for T in TS]
               + [(N, T, 1.0, True) for N in (4, 8, 64, 256) for T in (4, 8, 16)]           # chan_run_regs<T>
               + [(6, 3, 1.0, False), (7, 5, 1.0, False), (12, 2, 1.0, False), (1000, 2, 1.0, False),  # Bluestein
                  (512, 3, 1.0, False), (4096, 2, 1.0, False),                                 # radix, wide grids
                  (64, 33, 1.0, False), (8, 33, 1.0, False),                                   # above the fused limit
                  (64, 5, 2.0, False), (64, 5, 4.0, False), (64, 3, 64.0, False), (8, 4, 8.0, False)])  # oversampled

SYNTH_NS = [2, 3, 4, 5, 8, 64, 128, 256, 512]
# (N, T, no_fused)
SYNTH_SHAPES = ([(N, T, False) for N in SYNTH_NS for T in TS]
                + [(N, T, True) for N in SYNTH_NS for T in TS if fused_tpad(N, T)])

PFBARB_RATES = [0.1, 0.5, 0.768, 1.0, 1.6, 2.0, 2.37, 126.0]     # 126: the largest rate the plan accepts
DYADIC_RATES = [0.5, 1.6, 2.0]                                   # f32 delay = 1/rate is 2.0, 0.625, 0.5
# (arms, taps per arm, rate, periodic schedule).  pfb_kernel's branch (pfbarb.cu, b2s_pfbarb_exec): tile_in_smem when
# (sub_per_cta * sub-block + T + 2) * 8 B <= 64 KiB, arms_in_smem when arms * (T | 1) * 4 B <= 64 KiB.
#   32 x 5:    both in shared memory
#   64 x 300:  77 KiB of arms, tile in shared memory
#   4 x 6200:  a 66 KiB tile (2048 + 6202 items at rate 1), global memory
PFBARB_SHAPES = ([(32, 5, r, per) for r in PFBARB_RATES[:-1] for per in (True, False)]
                 + [(128, 3, PFBARB_RATES[-1], per) for per in (True, False)]
                 + [(7, 3, 0.768, True), (7, 1, 2.37, True)]
                 + [(64, 300, 1.0, True), (64, 300, 2.37, False), (4, 6200, 1.0, True), (4, 6200, 0.768, False)])
# Rates above the arm count: tau is negative when the output after a Boundary state advances it, floor(tau * N) < 0
# and the reference's `as usize` saturates it to arm 0.  The oracle's C cast does not (undefined; it wraps on x86-64),
# so these shapes are checked against ArbRef.  122 is the largest rate 32 arms accept (pfbarb_per_sample_max).
PFBARB_HIGH_SHAPES = [(32, 5, 33.0, True), (32, 5, 33.0, False), (32, 5, 122.0, True), (32, 5, 64.0, False),
                      (4, 3, 50.0, True), (1, 3, 20.0, True)]


def pfbarb_per_sample_max(rate, N):
    """pfbarb.cu's bound on the outputs of one input sample."""
    if np.float32(rate) <= N:
        return int(np.ceil(np.float32(rate))) + 1
    return int(np.ceil(float(np.float32(rate)) * (1.0 + 1.0 / N))) + 2


# ---- call sequences -------------------------------------------------------------------------------------------------
def drive(work, n_total, steps, drain_cap):
    """Calls work(pos, avail, cap) -> (consumed, produced, call_again, out) once per (avail, cap) of `steps` -- the call
    sees the next min(avail, n_total - pos) unconsumed items; avail may be a function of pos -- then with everything
    left and drain_cap (also the largest capacity) until a call does nothing.  Returns [(pos, avail, cap, (consumed, produced, call_again), out)]."""
    calls, pos = [], 0
    todo = list(steps)
    for _ in range(10000):
        if todo:
            avail, cap = todo.pop(0)
        else:
            avail, cap = n_total, drain_cap
        avail = max(0, min(avail(pos) if callable(avail) else avail, n_total - pos))
        cap = min(cap, drain_cap)
        c, p, ca, out = work(pos, avail, cap)
        calls.append((pos, avail, cap, (c, p, bool(ca)), out))
        pos += c
        if not todo and c == 0 and p == 0 and not ca:
            return calls
    raise AssertionError("drive: no end")


def _crint(a):
    return np.rint(a.real) + 1j * np.rint(a.imag)


# ---- channelizer ----------------------------------------------------------------------------------------------------
def chan_case(N, T, osr, seed, lim=LIM):
    """Taps of N*T integer values (the last arm zero padded when T > 1: ntaps = N*T - N//2), and the decimation."""
    rng = np.random.default_rng(seed)
    ntaps = N * T - (N // 2 if T > 1 else 0)
    return rng, int_taps(rng, ntaps, lim=lim), int(np.float32(N) / np.float32(osr))


def chan_vectors(N, T, D):
    """Output vectors a test input gives: past the first T-1 of a call and two fused tiles, or 40 past the vectors whose
    windows still hold start-up samples (N*T/D of them)."""
    return T + (2 * fused_ob(N) + 5 if fused_tpad(N, T) and D == N else 40 + 2 * N * T // D)


def chan_patterns(N, T, D):
    """{name: steps}.  ragged: 1 item, a cut inside the window fill, the rest of the fill (that call consumes nothing),
    T-1 vectors, one fused tile +- 1 after the T-1 generic ones, then the rest.  caps: capacities 0, 1, T-1, T, tile+1
    on the whole remaining input."""
    NT, ob = N * T, fused_ob(N)
    big = 1 << 40
    fill = [(1, big), (max(NT // 2 - 1, 0), big), (NT, big)]
    return {
        "all": [],
        "ragged": fill + [((T - 1) * D, big), ((T - 1 + ob + 1) * D, big), ((T - 1 + ob - 1) * D + D // 2, big)],
        "caps": [(NT, big)] + [(big, c) for c in (0, 1, max(T - 1, 0), T, ob + 1)],
    }


def chan_arms(y):
    """The arm outputs of each output vector: y [N, n] channel-major -> FFT_f64 over the channels / N, [N, n]."""
    y = np.asarray(y, np.complex128)
    return np.fft.fft(y, axis=0) / y.shape[0]


def chan_expect(y):
    """Expected values from the oracle's outputs y [N, p]: (finite mask [N, p], integer arms [N, p] of the vectors whose
    outputs are all finite, NaN elsewhere).  Asserts that the oracle's own recovery lands on integers."""
    fin = np.isfinite(y)
    a = np.full(y.shape, np.nan, np.complex128)
    cols = np.flatnonzero(fin.all(axis=0))
    if cols.size:
        r = chan_arms(y[:, cols])
        ri = _crint(r)
        err = float(np.max(np.abs(r - ri)))
        assert err < RECOVER_TOL, f"channelizer oracle arms are {err} from integers"
        a[:, cols] = ri
    return fin, a


def chan_run(N, taps, osr, x, steps):
    """The oracle through `steps` (drive()).  Each call's out is (y [N, p] float32, finite mask, integer arms)."""
    o = orc.PfbChannelizer(N, taps, osr)
    big = x.size // o.D + 8

    def work(pos, avail, cap):
        c, p, ca, y = o.work(x[pos:pos + avail], min(cap, big))
        return c, p, ca, (y,) + chan_expect(y)
    return drive(work, x.size, steps, big)


def chan_textbook(N, D, taps, pushed, n_out):
    """Steady state of the channelizer in float64: push c of the stream goes to window (N-1-c) mod N, so window w is the
    pushed stream decimated by N at a fixed phase; output o is formed after E = N*T + (o+1)*D pushes, and arm i (taps
    [i::N]) meets window (base + i + 1) mod N, base = (N-1-E) mod N, oldest sample first.  Returns the arm outputs
    [N (window), n_out] and a mask of the outputs whose windows hold no item of the start-up fill (c >= N*T)."""
    T = -(-len(taps) // N)
    arms = np.zeros((N, T))
    for i in range(N):
        a = np.asarray(taps[i::N], np.float64)
        arms[i, :a.size] = a
    P = np.asarray(pushed, np.complex128)
    out = np.zeros((N, n_out), np.complex128)
    ok = np.zeros(n_out, bool)
    for o in range(n_out):
        E = N * T + (o + 1) * D
        base = (N - 1 - E) % N
        oldest = E
        for i in range(N):
            b = (base + i + 1) % N
            r = (N - 1 - b) % N
            c_new = r + ((E - 1 - r) // N) * N
            idx = c_new - np.arange(T) * N                # j-th newest: tap j
            oldest = min(oldest, int(idx[-1]))
            out[b, o] = np.sum(P[idx] * arms[i]) if idx[-1] >= 0 else np.nan
        ok[o] = oldest >= N * T
    return out, ok


# ---- synthesizer ----------------------------------------------------------------------------------------------------
def synth_inputs(rng, N, nv, lim=2):
    """Channel-major inputs x [N, nv] complex64 whose un-normalised inverse DFTs are the integer vectors s [N, nv]
    (values in [-lim, lim]): x = FFT_f64(s) / N.  Returns (x, s)."""
    s = (rng.integers(-lim, lim + 1, (N, nv)) + 1j * rng.integers(-lim, lim + 1, (N, nv))).astype(np.complex128)
    return (np.fft.fft(s, axis=0) / N).astype(np.complex64), s


def synth_case(N, T, seed):
    rng = np.random.default_rng(seed)
    return rng, int_taps(rng, max(N * T - (N // 2 if T > 1 else 0), 1), lim=LIM)


def synth_vectors(N, T):
    """Input vectors of a test: past the fill, the generic lead and three fused tiles, or 40 steady vectors."""
    return T + (synth_lead(N, T) + 3 * fused_ob(N) + T + 3 if fused_tpad(N, T) else 40)


def synth_patterns(N, T):
    """{name: steps} in vectors and output items.  ragged: 1 vector, a cut inside the fill, the fill completing in the
    middle of a call, T-1 vectors, one fused tile +- 1 past the generic lead, then the rest.  caps: the fill, then
    output capacities 0, 1, N, N+1, 2N, 2N+1 and one tile + 1 (the loop runs while cap - produced > N)."""
    ob, lead = fused_ob(N), synth_lead(N, T)
    big = 1 << 40
    fill = [(1, big), (max(T // 2 - 1, 0), big), (T + 3, big)] if T > 1 else [(4, big)]
    return {
        "all": [],
        "ragged": fill + [(max(T - 1, 1), big), (lead + ob + 1, big), (lead + ob - 1, big)],
        "caps": [(T, N)] + [(big, c) for c in (0, 1, N, N + 1, 2 * N, 2 * N + 1, (ob + 1) * N + 1)],
    }


def synth_expect(out):
    """Expected values from the oracle's outputs: (finite mask, rint of the outputs).  Asserts that every finite
    oracle output is within RECOVER_TOL of an integer."""
    fin = np.isfinite(out)
    z = np.where(fin, _crint(np.where(fin, out, 0).astype(np.complex128)), np.nan)
    if fin.any():
        err = float(np.max(np.abs(out[fin].astype(np.complex128) - z[fin])))
        assert err < RECOVER_TOL, f"synthesizer oracle outputs are {err} from integers"
    return fin, z


def synth_run(N, taps, x, steps):
    """The oracle through `steps` (drive(), in vectors).  Each call's out is (out float32, finite mask, integers)."""
    o = orc.PfbSynthesizer(N, taps)
    big = (x.shape[1] + 2) * N

    def work(pos, avail, cap):
        c, p, y = o.work(x[:, pos:pos + avail], min(cap, big))
        return c, p, False, (y,) + synth_expect(y)
    return drive(work, x.shape[1], steps, big)


def synth_textbook(N, taps, s):
    """Steady state of the synthesizer in float64: spun sample s[w, v] enters window w, and output (v-T+1)*N + w is
    sum_j s[w, v-j] * taps[w + j*N].  Returned for v >= 2T-1 (the start-up fill writes its windows scattered), with the
    index of its first output."""
    T = -(-len(taps) // N)
    arms = np.zeros((N, T))
    for w in range(N):
        a = np.asarray(taps[w::N], np.float64)
        arms[w, :a.size] = a
    nv = s.shape[1]
    v0 = 2 * T - 1
    out = np.zeros((max(nv - v0, 0), N), np.complex128)
    for v in range(v0, nv):
        out[v - v0] = np.einsum("wj,wj->w", s[:, v - np.arange(T)], arms)
    return out.reshape(-1), (v0 - (T - 1)) * N


# ---- PfbArbResampler ------------------------------------------------------------------------------------------------
def pfbarb_case(N, T, rate, seed):
    """Taps, and an input of T fill samples plus enough steady samples for several CTAs of pfb_kernel."""
    rng = np.random.default_rng(seed)
    taps = int_taps(rng, N * T - (N // 2 if T > 1 else 0), lim=LIM)
    return taps, int_samples(rng, T + max(600, min(5000, int(20000 / rate))), True, lim=LIM)


def _arm_index(bf):
    """`bf.floor() as usize`: saturating, a negative floor gives arm 0."""
    return max(int(np.floor(bf)), 0)


def pfbarb_timing(rate, N, n):
    """The timing recurrence of arb_resampler.rs:132-188 in numpy float32 for n steady samples: per output (sample,
    arm of y0, mu, boundary), and per sample whether the Boundary state is pending after it."""
    f32 = np.float32
    delay, fN = f32(1.0) / f32(rate), f32(N)
    tau, mu, base, boundary = f32(0), f32(0), 0, False
    outs, pending = [], np.zeros(n, bool)

    def update():
        nonlocal tau, mu, base
        tau = f32(tau + delay)
        bf = f32(tau * fN)
        base = _arm_index(bf)
        mu = f32(bf - f32(base))
    for s in range(n):
        while base < N:
            if boundary:
                outs.append((s, N - 1, mu, True))
                update()
                boundary = False
            elif base == N - 1:
                boundary, base = True, N
            else:
                outs.append((s, base, mu, False))
                update()
        tau = f32(tau - f32(1.0))
        base -= N
        pending[s] = boundary
    return outs, pending


def pfbarb_textbook(rate, N, taps, x):
    """Outputs of the steady state in float64: output (s, b, mu) is (1-mu)*arm_b . w(s) + mu*arm_{b+1} . w(s) with w(s)
    the T samples ending at x[T + s] (Boundary: arm N-1 on w(s-1), arm 0 on w(s)); exact in f32 when mu is dyadic.
    Returns (all outputs, mask of those whose windows hold no sample of the start-up fill)."""
    T = -(-len(taps) // N)
    arms = np.zeros((N, T))
    for i in range(N):
        a = np.asarray(taps[i::N], np.float64)
        arms[i, :a.size] = a
    xx = np.asarray(x, np.complex128)
    outs, _ = pfbarb_timing(rate, N, xx.size - T)

    def dot(b, s):
        k = T + s                                      # newest sample of the window
        return np.sum(xx[k - np.arange(T)] * arms[b]) if k - T + 1 >= 0 else np.nan
    y = np.zeros(len(outs), np.complex128)
    ok = np.zeros(len(outs), bool)
    for k, (s, b, mu, bnd) in enumerate(outs):
        mu = float(mu)
        if bnd:
            y[k] = (1 - mu) * dot(N - 1, s - 1) + mu * dot(0, s)
        else:
            y[k] = (1 - mu) * dot(b, s) + mu * dot(b + 1, s)
        ok[k] = s - 1 >= T
    return y, ok


class ArbRef:
    """PfbArbResampler's Kernel::work (arb_resampler.rs:90-231) restated in numpy: the WindowBuffer with its scattered
    fill, the float32 timing recurrence with the saturating arm index, the arm dots (exact integers here, computed in
    float64) and the blend (1-mu)*y0 + mu*y1 in separately rounded float32 operations.  Same interface as the oracle's
    work(); equal to it bit for bit wherever rate <= arms (test_pfb_exact_reference.py)."""

    def __init__(self, rate, taps, N):
        f32 = np.float32
        self.N, self.rate = N, f32(rate)
        self.T = T = int(np.ceil(f32(len(taps)) / f32(N)))
        self.rev = np.zeros((N, T))                     # arm i reversed: rev[i, t] = arm_i[T-1-t]
        for i in range(N):
            a = np.asarray(taps[i::N], np.float64)
            self.rev[i, T - a.size:] = a[::-1]
        self.circ = np.zeros(T, np.complex128)
        self.start, self.missing = 0, T
        self.delay, self.fN = f32(1.0) / f32(rate), f32(N)
        self.tau, self.mu, self.base, self.boundary = f32(0), f32(0), 0, False
        self.buff0 = 0j

    def _push(self, v):
        T = self.T
        self.circ[(self.start - self.missing) % T] = v
        self.missing = max(self.missing - 1, 0)
        self.start = (self.start + 1) % T

    def _update(self):
        f32 = np.float32
        self.tau = f32(self.tau + self.delay)
        bf = f32(self.tau * self.fN)
        self.base = _arm_index(bf)
        self.mu = f32(bf - f32(self.base))

    def _blend(self, y0, y1):
        f32 = np.float32
        a = f32(f32(1.0) - self.mu)
        re = f32(f32(a * f32(y0.real)) + f32(self.mu * f32(y1.real)))
        im = f32(f32(a * f32(y0.imag)) + f32(self.mu * f32(y1.imag)))
        return complex(re, im)

    def work(self, x, cap):
        x = np.asarray(x, np.complex128)
        if self.missing:
            c = min(self.missing, x.size)
            for v in x[:c]:
                self._push(v)
            return c, 0, x.size - c > 0, np.zeros(0, np.complex64)
        n = min(x.size, int(np.float32(cap) / self.rate))
        out, N = [], self.N
        for v in x[:n]:
            self._push(v)
            win = np.concatenate((self.circ[self.start:], self.circ[:self.start]))   # get_as_slice, oldest first
            while self.base < N:
                if self.boundary:
                    out.append(self._blend(self.buff0, win @ self.rev[0]))
                    self._update()
                    self.boundary = False
                elif self.base == N - 1:
                    self.buff0 = win @ self.rev[N - 1]
                    self.boundary, self.base = True, N
                else:
                    out.append(self._blend(win @ self.rev[self.base], win @ self.rev[self.base + 1]))
                    self._update()
            self.tau = np.float32(self.tau - np.float32(1.0))
            self.base -= N
        return n, len(out), False, np.array(out, np.complex64)


def _arb_work(o, x, cap):
    """orc.PfbArb.work with an output buffer that holds whatever the schedule produces, also beyond `cap`."""
    import ctypes as C
    if isinstance(o, ArbRef):
        return o.work(x, cap)
    xi = np.ascontiguousarray(x, np.complex64)
    n = min(xi.size, int(np.float32(cap) / o.rate))
    out = np.zeros(n * (int(np.ceil(o.rate)) + 1) + 16, np.complex64)
    c, p, ca = C.c_size_t(0), C.c_size_t(0), C.c_int(0)
    f32p = C.POINTER(C.c_float)
    orc.lib().orc_pfbarb_work(o._h, xi.view(np.float32).ctypes.data_as(f32p), xi.size,
                              out.view(np.float32).ctypes.data_as(f32p), cap, C.byref(c), C.byref(p), C.byref(ca))
    return c.value, p.value, bool(ca.value), out[:p.value].copy()


def pfbarb_run(rate, N, taps, x, steps, ref=None):
    """The oracle -- ArbRef where rate > N, or where ref=ArbRef -- through `steps` (drive()).  A call whose schedule
    would produce more than its capacity (the
    reference overruns its slice there; the device refuses it with B2S_ESTATE and commits nothing) is returned with
    counts None and out None, and the oracle is rebuilt and replayed to the state before it.  (No shape and capacity
    pattern here reaches that, the Boundary-pending starts of the caps pattern and the rates above the arm count
    included: the count rule n = cap / rate keeps the schedule within the slice.  The branch stays so that the tests
    check B2S_ESTATE if a schedule ever overruns.)  Each accepted call's
    out is (out complex64, finite mask)."""
    accepted = []
    make = ref or (ArbRef if np.float32(rate) > N else orc.PfbArb)
    state = {"o": make(rate, taps, N)}
    big = int(np.ceil(x.size * rate)) + 64

    def work(pos, avail, cap):
        cap = min(cap, big)
        c, p, ca, y = _arb_work(state["o"], x[pos:pos + avail], cap)
        if p > cap:
            o = make(rate, taps, N)
            for (ps, av, cp) in accepted:
                _arb_work(o, x[ps:ps + av], cp)
            state["o"] = o
            return 0, 0, True, None                   # (call_again: the driver keeps going)
        accepted.append((pos, avail, cap))
        return c, p, ca, (y, np.isfinite(y))
    calls = drive(work, x.size, steps, big)
    return [(pos, av, cp, None if out is None else cnt, out) for (pos, av, cp, cnt, out) in calls]


def pfbarb_patterns(rate, N, T, n):
    """{name: steps}.  ragged: 1 item, a cut inside the fill, the rest of the fill, calls that end while the Boundary
    state is pending, then the rest.  caps: the fill, then capacities 0, 1, T-1, T, 2049 and 2..13, 2*rate + 1, each on
    a call that starts with a Boundary output pending (the first sample then produces one output more), so that some
    of them make the schedule overrun the slice (pfbarb_run)."""
    big = 1 << 40
    _, pending = pfbarb_timing(rate, N, min(n, 4000))
    cuts = np.flatnonzero(pending)
    ragged = [(1, big), (max(T // 2 - 1, 0), big), (big, big)]  # the fill call consumes only the missing samples
    done = 0                                           # steady samples consumed so far
    for s in cuts[cuts >= 2][:3]:
        ragged.append((int(s) + 1 - done, big))         # the call ends right after sample s
        done = int(s) + 1

    def to_pending(pos):                               # up to the next sample that leaves the Boundary state pending
        nxt = cuts[cuts >= pos - T]
        return int(nxt[0]) + 1 - (pos - T) if nxt.size else 0
    caps = [(T, big)]
    for c in (0, 1, max(T - 1, 0), T, 2049, *range(2, 14), 2 * int(rate) + 1):
        caps += [(to_pending, big), (big, c)]
    return {"all": [], "ragged": ragged, "caps": caps}
