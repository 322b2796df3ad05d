"""The fused spectrum pipe (spectrum.cu, blocks.SpectrumPipe) bin by bin, against a float64 evaluation of the average.

The pipe computes, per bin, the recurrence  avg_k = a*avg_{k-1} + d*t_k  (a = 1-d in f32, t_k = |X_k|^2, skipped when
non-finite) as a blocked scan: a local chain per group of C frames from zero, a scan that composes the groups' affine
maps  x -> final_g + a^C x, and a fix-up that adds  a^k * carry_g  to every emitted row.  Its values are therefore not
the sequential f32 recurrence's bits, and a gate relative to the largest average would let weak bins be wrong by
percents.  The tests here separate the two stages:

* the periodogram t is taken from the pipe itself: SpectrumPipe(N, decay=1, history=1) emits exactly  0*avg + 1*t = t
  (the fix-up weights are 0), and the FFT and the squaring depend on neither decay, history nor grouping;
* the average is judged per emitted value of every bin against V, a float64 evaluation of the same recurrence on that
  t, with a running bound B on the error of the sequential f32 recurrence (see ``Bound``);
* the transform is judged per frame, normwise, against numpy's complex128 FFT (a bin's power can be arbitrarily close
  to 0 while the FFT's rounding error is bounded per frame, so a per-bin relative gate is only sound on the average).

The CPU half emulates the blocked scan in numpy and shows that the gate fails a pipe whose fix-up power index is off
by one, which drops one group's carry, or which swaps the scan's A and A_last, and that it fails f32 weights a^k once
they underflow (a loud tone followed by silence)."""
import ctypes
import math

import numpy as np
import pytest
from scipy.signal import lfilter

import oracle as orc

U = 2.0 ** -24                       # unit roundoff of f32
ETA = 2.0 ** -150                    # absolute rounding error of a result in f32's subnormal range
U2 = 2 * U + U * U                   # one multiply, then one add, of the sequential recurrence
SIZES = [1 << k for k in range(5, 14)]
MAX_CTAS_PER_SM = 8                  # 2048 threads per SM / 256 threads per CTA: an upper bound on occupancy


def coeffs(decay):
    """(a, d) exactly as the pipe and the oracle hold them: d = f32(decay), a = 1 - d in f32."""
    d = np.float32(decay)
    return float(np.float32(1.0) - d), float(d)


def transforms_per_cta(n):
    """fft_geom(log2 n, 256).fpb: one radix-16 butterfly per thread, at most the whole 256-thread CTA per transform."""
    return 256 // min(256, max(1, n // 16))


class Bound:
    """V_k = a V_{k-1} + d t_k in float64 (t_k = 0 for skipped frames), and a bound B_k on |avg_k - V_k| for the
    sequential f32 recurrence avg_k = fl(fl(a avg_{k-1}) + fl(d t_k)).

    One step rounds twice, each time by at most a relative u or, in the subnormal range, an absolute eta (an add whose
    result is subnormal is exact), so its local error is at most U2 (a|avg_{k-1}| + d t_k) + 2 eta
    <= U2 V_k + U2 a |avg_{k-1} - V_{k-1}| + 2 eta.  Hence  B_k = a (1 + U2) B_{k-1} + U2 V_k + 2 eta.
    Both are first-order recurrences along the frame axis, evaluated by lfilter with the state carried across calls;
    float64's own rounding of V (relative ~2^-53 / (1 - a)) is far below B."""

    def __init__(self, n, decay):
        self.a, self.d = coeffs(decay)
        self.n = n
        self.reset()

    def reset(self):
        self.zv = np.zeros((self.n, 1))
        self.zb = np.zeros((self.n, 1))

    def advance(self, t):
        """t: (frames, n) with skipped frames zeroed -> (V, B), (frames, n) float64.  (lfilter runs along the last,
        contiguous axis: bins x frames.)"""
        x = np.ascontiguousarray(t.T, dtype=np.float64)
        x *= self.d
        V, self.zv = lfilter([1.0], [1.0, -self.a], x, axis=-1, zi=self.zv)
        x = U2 * V
        x += 2 * ETA
        B, self.zb = lfilter([1.0], [1.0, -self.a * (1 + U2)], x, axis=-1, zi=self.zb)
        return V.T, B.T


def pipe_limit(V, B):
    """What the blocked scan may differ from V by.  Its value at frame k of group g is
    fl(w_k * carry_g + L_{g,k}), L the group's local chain from zero:
    * the local chains run the reference's two roundings per frame, and the carries are composed from the local
      chains' final states, so their rounding errors together are within B (B is linear: the bound of a local chain
      from zero plus a^k times the bound at the group's start);
    * the scan rounds once per group where it composes a segment (one fma) and once where it walks it (one fma);
      each of those is at most u times the state at the group's end, V_end, which is at most half of what B itself
      adds at the group's last frame (U2 V_end): a second B;
    * the carry is stored in f32 (u V), the weight a^k is rounded (u V while a^k is a normal f32, 2^-53 V in f64),
      the fix-up's fma rounds once (u V); the fourth u V takes the second-order terms.  Each of the carry, the
      weighted carry and the fix-up can be subnormal: the 4 eta."""
    return 2 * B + 4 * U * V + 4 * ETA


class Gate:
    """Per emitted value of every bin: the f32 oracle within B of V (the bound is real), the pipe within
    ``pipe_limit``.  Keeps the largest observed error-to-bound ratios."""

    def __init__(self):
        self.ref_ratio = 0.0
        self.pipe_ratio = 0.0
        self.values = 0

    def check(self, got, ref, V, B, what=""):
        got = got.astype(np.float64)
        ref = ref.astype(np.float64)
        assert np.all(np.isfinite(got)) and np.all(np.isfinite(ref)), what
        rerr = np.abs(ref - V)
        assert np.all(rerr <= B), (what, "oracle outside its bound", float(np.max(rerr / B)))
        lim = pipe_limit(V, B)
        err = np.abs(got - V)
        bad = err > lim
        if np.any(bad):
            r, b = np.argwhere(bad)[0]
            raise AssertionError(f"{what}: {int(bad.sum())} values outside the bound; first at row {r} bin {b}: "
                                 f"got {got[r, b]!r} V {V[r, b]!r} bound {lim[r, b]!r}")
        self.ref_ratio = max(self.ref_ratio, float(np.max(rerr / B, initial=0.0)))
        self.pipe_ratio = max(self.pipe_ratio, float(np.max(err / lim, initial=0.0)))
        self.values += got.size


def emitted_mask(i0, frames, history):
    """Which of `frames` frames emit a row, with i0 frames since the last emission (moving_avg.rs: self.i)."""
    return (i0 + np.arange(frames) + 1) % history == 0


# ------------------------------------------------------------------------------------------------ CPU emulation


def _fma32(a, b, c):
    """fmaf on f32 operands: the product is exact in float64; the sum can round twice (irrelevant next to the gate)."""
    return (np.float64(a) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def emulate_pipe(t, skip, decay, history, calls, g_target, weights=np.float64, mutate=None):
    """b2s_spectrum_exec over the periodogram frames t (frames, n) f32, skip: (frames,) bool, in calls of `calls`
    frames each, with C = max(4, ceil(frames / g_target)) as the host picks it.  ``weights=np.float32`` is the scan
    and fix-up with f32 weights a^k, a^C and f32 segment products; ``np.float64`` holds them, the scan's states and
    the fix-up's product in float64.  ``mutate``: None, "pow_index" (fix-up weight a^(k-1)), "drop_carry" (the
    carry of one group of the first multi-group call is lost), "a_last" (the scan swaps A and A_last).
    Returns the emitted rows (rows, n) f32 and their frame indices."""
    n = t.shape[1]
    a32 = np.float32(1.0) - np.float32(decay)
    d32 = np.float32(decay)
    a64 = float(a32)
    f32w = weights is np.float32
    state = np.zeros(n, np.float32)
    i, pos, rows, at = 0, 0, [], []
    dropped = False
    for F in calls:
        C = max(4, -(-F // g_target))
        G = -(-F // C)
        c_last = F - (G - 1) * C
        tp = np.zeros((G * C, n), np.float32)
        tp[:F] = t[pos:pos + F]
        sk = np.zeros(G * C, bool)
        sk[:F] = skip[pos:pos + F]
        tp, sk = tp.reshape(G, C, n), sk.reshape(G, C)
        active = (np.arange(G)[:, None] * C + np.arange(C)[None, :]) < F
        avg = np.zeros((G, n), np.float32)
        loc = np.zeros((G, C, n), np.float32)
        for c in range(C):                       # local chains, the reference's un-fused order
            dec = a32 * avg
            new = np.where(sk[:, c, None], dec, dec + d32 * tp[:, c])
            avg = np.where(active[:, c, None], new, avg)
            loc[:, c] = avg
        fin = avg
        A, A_last = a64 ** C, a64 ** c_last
        if f32w:
            A, A_last = np.float32(A), np.float32(A_last)
        if mutate == "a_last":
            A, A_last = A_last, A
        Ag = [A] * (G - 1) + [A_last]
        per = -(-G // 32)
        segs = [(s * per, min(s * per + per, G)) for s in range(32) if s * per < G]
        carry = np.zeros((G, n), np.float32)
        if f32w:
            x = state.copy()
            for g0, g1 in segs:
                L, M = np.zeros(n, np.float32), np.float32(1.0)
                for g in range(g0, g1):
                    L = _fma32(Ag[g], L, fin[g])
                    M = np.float32(M * Ag[g])
                xs = x
                x = _fma32(M, x, L)
                for g in range(g0, g1):          # the walk from the segment's known start state
                    carry[g] = xs
                    xs = _fma32(Ag[g], xs, fin[g])
            state = x
        else:
            x = state.astype(np.float64)
            for g0, g1 in segs:
                L, M = np.zeros(n), 1.0
                for g in range(g0, g1):
                    L = Ag[g] * L + fin[g]
                    M *= Ag[g]
                xs = x
                x = M * x + L
                for g in range(g0, g1):
                    carry[g] = xs.astype(np.float32)
                    xs = Ag[g] * xs + fin[g]
            state = x.astype(np.float32)
        if mutate == "drop_carry" and not dropped and G > 2:
            carry[G // 2] = 0.0
            dropped = True
        pw = np.array([a64 ** k for k in range(C + 1)])
        if f32w:
            pw = pw.astype(np.float32)
        for fs in np.nonzero(emitted_mask(i, F, history))[0]:
            g = fs // C
            k = fs - g * C + 1
            w = pw[k - 1] if mutate == "pow_index" else pw[k]
            if f32w:
                rows.append(_fma32(w, carry[g], loc[g, k - 1]))
            else:
                rows.append((w * carry[g].astype(np.float64) + loc[g, k - 1]).astype(np.float32))
            at.append(pos + fs)
        i = (i + F) % history
        pos += F
    return np.array(rows, np.float32).reshape(-1, n), np.array(at, np.int64)


def gate_emulation(t, skip, decay, history, calls, g_target, **kw):
    got, at = emulate_pipe(t, skip, decay, history, calls, g_target, **kw)
    tz = np.where(skip[:, None], np.float32(0.0), t)
    V, B = Bound(t.shape[1], decay).advance(tz[:sum(calls)])
    ref = orc.MovingAvg(t.shape[1], decay, history)
    tn = np.where(skip[:, None], np.float32(np.nan), t)
    _, _, want = ref.work(tn[:sum(calls)].ravel(), tn.size)
    gate = Gate()
    gate.check(got, want.reshape(-1, t.shape[1]), V[at], B[at])
    return gate


def _random_stream(rng, frames, n):
    t = (rng.exponential(1.0, (frames, n)) * np.where(np.arange(n) % 5 == 0, 1e4, 1.0)).astype(np.float32)
    t[10:13] = 0.0                                        # all-zero frames
    skip = np.zeros(frames, bool)
    skip[[4, 40, 97]] = True
    return t, skip


CALLS = [7, 50, 1000, 3, 413]                             # g_target 80: C = 4, 4, 13 (77 groups, partial last), 4, 6


@pytest.mark.parametrize("decay,history", [(0.01, 1), (0.1, 3), (0.25, 2), (0.5, 7), (0.9, 1)])
@pytest.mark.parametrize("weights", [np.float32, np.float64], ids=["f32_weights", "f64_weights"])
def test_emulated_scan_within_bound(rng, decay, history, weights):
    t, skip = _random_stream(rng, sum(CALLS), 16)
    g = gate_emulation(t, skip, decay, history, CALLS, 80, weights=weights)
    print(f"decay {decay} history {history} {weights.__name__}: {g.values} values, "
          f"oracle/B {g.ref_ratio:.3g}, emulated pipe/limit {g.pipe_ratio:.3g}")


@pytest.mark.parametrize("mutate", ["pow_index", "drop_carry", "a_last"])
@pytest.mark.parametrize("decay", [0.1, 0.5])
def test_emulated_scan_mutations_fail_the_gate(rng, mutate, decay):
    t, skip = _random_stream(rng, sum(CALLS), 16)
    with pytest.raises(AssertionError, match="outside the bound"):
        gate_emulation(t, skip, decay, 1, CALLS, 80, mutate=mutate)


def _tone_then_silence(n, tone_frames, frames):
    t = np.zeros((frames, n), np.float32)
    t[:tone_frames, 0] = 1e30
    t[:tone_frames, 1] = 1e12
    t[:tone_frames, 2] = 4e7
    return t, np.zeros(frames, bool)


@pytest.mark.parametrize("decay", [0.5, 0.9])
def test_emulated_silence_after_tone_needs_f64_weights(decay):
    """A loud bin followed by silence, in a call long enough that C > 150: the average decays through f32's
    subnormal range long after a^k and a^C have underflowed there.  f32 weights lose it; float64 weights keep it."""
    t, skip = _tone_then_silence(4, 64, 64 + 800)
    calls = [64, 800]                                      # g_target 4: the long call has C = 200
    gate_emulation(t, skip, decay, 1, calls, 4, weights=np.float64)
    with pytest.raises(AssertionError, match="outside the bound"):
        gate_emulation(t, skip, decay, 1, calls, 4, weights=np.float32)


# ------------------------------------------------------------------------------------------------ device


def _device_stream(n_items, N, seed, tone_amp=30.0, tone_bin_frac=0.2):
    """Unit complex noise plus a strong tone on the device, so that weak bins are judged on their own."""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n_items, dtype=torch.complex64, device="cuda", generator=gen)
    k = torch.arange(n_items, dtype=torch.float64, device="cuda")
    ph = 2 * math.pi * torch.remainder(k * tone_bin_frac, 1.0)
    x += (tone_amp * torch.exp(1j * ph)).to(torch.complex64)
    return x


class Run:
    """A SpectrumPipe under test fed call by call, with the oracle MovingAvg and the float64 Bound on the same
    periodogram (taken from a decay-1 pipe of the same shift)."""

    CHUNK = 1 << 22                                       # values per gate evaluation

    def __init__(self, N, decay, history, shift, log10_scales=()):
        from futuresdr_b200.blocks import SpectrumPipe
        self.N, self.decay, self.h, self.shift = N, decay, history, shift
        self.blk = SpectrumPipe(N, decay, history, fft_shift=shift)
        self.logs = [(k, SpectrumPipe(N, decay, history, fft_shift=shift, log10_scale=k)) for k in log10_scales]
        self.per = SpectrumPipe(N, 1.0, 1, fft_shift=shift)
        self.ref = orc.MovingAvg(N, decay, history)
        self.bound = Bound(N, decay)
        self.gate = Gate()
        self.i = 0
        self.outputs = []
        self.log_outputs = {k: [] for k, _ in self.logs}

    def periodogram(self, x):
        import torch
        out = torch.empty(x.numel(), dtype=torch.float32, device="cuda")
        assert self.per.process(x, out) == (x.numel(), x.numel())
        return out.cpu().numpy().reshape(-1, self.N)

    def reset(self):
        self.blk.reset()
        for _, b in self.logs:
            b.reset()
        self.ref = orc.MovingAvg(self.N, self.decay, self.h)
        self.bound.reset()
        self.i = 0

    def call(self, x, cap, poisoned=()):
        """One process() call on the device slice x with an output capacity of cap floats; poisoned: indices (within
        x) of the frames holding a non-finite sample."""
        import torch
        N = self.N
        F = x.numel() // N
        t = self.periodogram(x[:F * N]) if F else np.zeros((0, N), np.float32)
        skip = np.zeros(F, bool)
        for f in poisoned:
            if f < F:
                _, X = orc.fft_block(x[f * N:(f + 1) * N].cpu().numpy(), N, fft_shift=self.shift)
                assert not np.any(np.isfinite(orc.norm_sqr(X))), "a poisoned frame must be non-finite in every bin"
                assert not np.any(t[f]), "a non-finite frame shows as 0 in the decay-1 pipe"
                skip[f] = True
        c0, p0, want = self.ref.work(np.where(skip[:, None], np.float32(np.nan), t).ravel(), cap)
        out = torch.zeros(max(cap, 1), dtype=torch.float32, device="cuda")[:cap]
        c, p = self.blk.process(x, out)
        for k, b in self.logs:
            lo = torch.zeros(max(cap, 1), dtype=torch.float32, device="cuda")[:cap]
            assert b.process(x, lo) == (c, p)
            self.log_outputs[k].append(lo[:p].cpu().numpy())
        assert (c, p) == (c0, p0), (F, cap, c, p, c0, p0)
        got = out[:p].cpu().numpy().reshape(-1, N)
        self.outputs.append(got.ravel())
        want = want.reshape(-1, N)
        Fc = c // N
        emit = emitted_mask(self.i, Fc, self.h)
        assert int(emit.sum()) == got.shape[0]
        tz = np.where(skip[:Fc, None], np.float32(0.0), t[:Fc])
        row = 0
        step = max(1, self.CHUNK // N)
        for f0 in range(0, Fc, step):
            V, B = self.bound.advance(tz[f0:f0 + step])
            e = emit[f0:f0 + step]
            r = int(e.sum())
            self.gate.check(got[row:row + r], want[row:row + r], V[e], B[e],
                            f"N {N} decay {self.decay} history {self.h} call of {F} frames")
            row += r
        self.i = (self.i + Fc) % self.h
        return c, p


def _feed(run, x, plan, poisoned=()):
    """Feeds x to run in the (items, capacity) steps of plan; poisoned: global frame indices."""
    pos = 0
    for step, cap in plan:
        seg = x[pos:pos + min(step, x.numel() - pos)]
        f0 = pos // run.N
        c, _ = run.call(seg, cap, [f - f0 for f in poisoned if f >= f0])
        pos += c
    return pos


def _long_frames(N):
    """Frames of a call that gives C >= 8 and more than 64 groups at any occupancy up to 8 CTAs per SM."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 8 * sms * MAX_CTAS_PER_SM * transforms_per_cta(N) + 13, sms


# N -> (decay, history, fft_shift): every size, with and without shift, every decay and history between them
STREAM_CASES = [(32, 0.0, 1, True), (64, 1e-3, 2, False), (128, 0.01, 3, True), (256, 0.1, 7, False),
                (512, 0.25, 257, True), (1024, 0.5, 1, False), (2048, 0.9, 2, True), (4096, 1.0, 3, False),
                (8192, 0.1, 7, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,decay,history,shift", STREAM_CASES)
def test_fused_spectrum_bins_long_and_ragged_calls(N, decay, history, shift):
    """Ragged short calls (output capacities below one row, a partial last group, idle transform slots), then one
    call long enough for C >= 8 and > 64 groups (d_pow and d_final regrow), then short calls again.  Noise plus a
    strong tone, all-zero frames, non-finite frames at group boundaries."""
    import torch
    L, sms = _long_frames(N)
    short1 = [(N * 7 + 5, N), (N * 50, N * 3), (N - 1, N * 4), (N * 3, 0), (N * 13, N * 1000)]
    short2 = [(N * 9 + 1, N * 2), (N * 5, N * 1000), (N * 11, N * 1000)]
    f_long = 7 + 50 + 13                                  # frames the first calls consume at most
    frames = f_long + L + 25
    x = _device_stream(frames * N, N, seed=N)
    x[:4 * N] = 0                                         # all-zero frames at the start
    mid = f_long + L // 2
    x[mid * N:(mid + 3) * N] = 0                          # and inside the long call
    run = Run(N, decay, history, shift)
    pos = _feed(run, x[:f_long * N], short1)              # the first calls consume fewer frames than offered
    f0 = pos // N
    # a group boundary of the long call at every occupancy it could run at, and the first frame of a short call
    cand = {f0}
    for res in range(1, MAX_CTAS_PER_SM + 1):
        C = max(4, -(-L // (sms * res * transforms_per_cta(N))))
        cand |= {f0 + C, f0 + C - 1, f0 + 2 * C}
    poisoned = sorted(cand | {f0 + L + 4})
    xp = x.clone()
    for f in poisoned:
        xp[f * N + 3] = complex(float("inf"), 0.0)
    plan = [(L * N, (L // history + 2) * N)] + short2
    pos += _feed(run, xp[pos:], plan, [f - f0 for f in poisoned])
    assert pos // N >= f0 + L + 16
    print(f"N {N} decay {decay} history {history} shift {shift}: {run.gate.values} values, largest oracle/B "
          f"{run.gate.ref_ratio:.3g}, pipe/limit {run.gate.pipe_ratio:.3g}")
    del x, xp
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_fused_spectrum_bins_silence_after_tone():
    """A loud bin (|X|^2 ~ 1e30 and its leakage) then silence, in a call long enough that a^C and the fix-up weights
    a^k underflow in f32 while a^k * carry is still a normal float: decay 0.5 needs C > 150, decay 0.9 C > 45.  At
    N = 8192 a CTA takes 132 KiB of shared memory, one per SM, so C = ceil(frames / SMs)."""
    import torch
    N = 8192
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tone = 64
    x = torch.zeros((tone + 152 * sms + 5) * N, dtype=torch.complex64, device="cuda")
    k = torch.arange(tone * N, dtype=torch.float64, device="cuda")
    x[:tone * N] = (1.2e11 * torch.exp(2j * math.pi * torch.remainder(k * 0.25, 1.0))).to(torch.complex64)
    for decay, history, C in ((0.5, 1, 152), (0.9, 2, 47)):
        quiet = C * sms - 3                               # C groups of frames, the last one partial
        run = Run(N, decay, history, True)
        run.call(x[:tone * N], tone * N)
        run.call(x[tone * N:(tone + quiet) * N], quiet * N)
        print(f"decay {decay}: {run.gate.values} values, largest oracle/B {run.gate.ref_ratio:.3g}, "
              f"pipe/limit {run.gate.pipe_ratio:.3g}")
        del run
    del x
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_fused_spectrum_reset_and_carried_state():
    """State carried across calls (the gate runs one recurrence over the whole stream), and reset() mid-stream equal
    to a fresh block bit for bit."""
    from futuresdr_b200.blocks import SpectrumPipe
    import torch
    N, decay, history = 256, 0.1, 3
    x = _device_stream(N * 400, N, seed=7)
    run = Run(N, decay, history, True)
    plan = [(N * 40 + 3, N * 1000), (N * 11, N * 2), (N * 60, N * 1000)]
    pos = _feed(run, x, plan)
    run.reset()
    fresh = SpectrumPipe(N, decay, history)
    for step, cap in [(N * 33, N * 1000), (N * 50, N * 5), (N * 90, N * 1000)]:
        seg = x[pos:pos + step]
        o = torch.zeros(cap, dtype=torch.float32, device="cuda")
        c, p = fresh.process(seg, o)
        assert run.call(seg, cap) == (c, p)
        assert np.array_equal(run.outputs[-1], o[:p].cpu().numpy())
        pos += c


@pytest.mark.gpu
def test_fused_spectrum_log10_per_value():
    """k*log10 of the pipe's own linear output: zero frames (-inf dB, times the sign of k), a loud tone, then silence
    that takes the average through f32's subnormal range (finite dB: the build does not flush to zero)."""
    import torch
    N, decay, history = 1024, 0.9, 1
    frames = 8 + 16 + 120
    x = torch.zeros(frames * N, dtype=torch.complex64, device="cuda")
    x[8 * N:24 * N] = _device_stream(16 * N, N, seed=3)
    scales = (10.0, -20.0, 3.5)
    run = Run(N, decay, history, True, log10_scales=scales)
    _feed(run, x, [(N * 5 + 1, N * 2), (N * 30, N * 1000), (N * 7, N * 3), (10 ** 9, N * 1000)])
    lin = np.concatenate(run.outputs)
    assert np.any(lin == 0) and np.any((lin > 0) & (lin < np.finfo(np.float32).tiny))
    with np.errstate(divide="ignore"):
        l10 = np.log10(lin.astype(np.float64))
    for k in scales:
        db = np.concatenate(run.log_outputs[k])
        assert db.shape == lin.shape
        zero = lin == 0
        assert np.all(db[zero] == np.float32(k) * np.float32(-np.inf))
        assert np.all(np.isfinite(db[~zero]))
        exact = k * l10[~zero]
        # log10f within 2 ulp of log10, then the multiply by k rounds once
        tol = abs(k) * 2 * np.spacing(np.abs(l10[~zero]).astype(np.float32)).astype(np.float64) \
            + 0.5 * np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
        err = np.abs(db[~zero].astype(np.float64) - exact)
        assert np.all(err <= tol), (k, float(np.max(err / tol)))


@pytest.mark.gpu
@pytest.mark.parametrize("N", SIZES)
def test_fused_spectrum_transform_stage(rng, N):
    """The decay-1 periodogram per frame against numpy's complex128 FFT, normwise (Higham, Accuracy and Stability
    of Numerical Algorithms, Thm 24.2: ||fl(FFT x) - FFT x|| <= log2(N) eta / (1 - log2(N) eta) ||FFT x||,
    eta = mu + gamma_4 (sqrt 2 + mu)); fft_shift=True equal to fft_shift=False rolled by N/2, bit for bit; and equal to
    the fused square fma(x, x, y*y) of the Fft block's output, which runs the same passes, plan and twiddle table."""
    import torch
    from futuresdr_b200.blocks import Fft, FftDirection, SpectrumPipe
    frames = 3 * transforms_per_cta(N) + 5                # idle transform slots in the last CTA
    x = (rng.standard_normal(N * frames) + 1j * rng.standard_normal(N * frames)).astype(np.complex64)
    x += (3 * np.exp(2j * np.pi * 0.2 * np.arange(x.size))).astype(np.complex64)
    xd = torch.from_numpy(x).cuda()
    P = {}
    for shift in (False, True):
        o = torch.empty(x.size, dtype=torch.float32, device="cuda")
        assert SpectrumPipe(N, 1.0, 1, fft_shift=shift).process(xd, o) == (x.size, x.size)
        P[shift] = o.cpu().numpy().reshape(frames, N)
    assert np.array_equal(P[True], np.roll(P[False], N // 2, axis=1))
    # normwise per frame.  mu bounds the relative error of every twiddle the passes apply: the table entry (u) raised
    # to at most the 15th power by the product tree of apply_twiddles (15 u), plus its at most 4 complex multiplies
    # (sqrt 2 gamma_2 each); the radix-16/8/4 DFTs' own rotations are within that.
    X = np.fft.fft(x.reshape(frames, N).astype(np.complex128), axis=1)
    g4 = 4 * U / (1 - 4 * U)
    mu = 15 * U + 4 * math.sqrt(2) * 2 * U / (1 - 2 * U)
    eta = mu + g4 * (math.sqrt(2) + mu)
    lg = math.log2(N)
    rel_fft = lg * eta / (1 - lg * eta)
    # |X|^2 = fma(x, x, fl(y*y)) is within (2u + u^2) |X|^2, so its square root within u (1 + u) |X|
    rel = rel_fft + U * (1 + U) * (1 + rel_fft)
    err = np.linalg.norm(np.sqrt(P[False].astype(np.float64)) - np.abs(X), axis=1)
    ratio = err / (rel * np.linalg.norm(X, axis=1))
    assert np.all(ratio <= 1.0), float(np.max(ratio))
    # the Fft block's output, squared on the host as the pipe's kernel squares it
    Y = torch.empty_like(xd)
    assert Fft.with_options(N, FftDirection.Forward, False, None).transform(xd, Y) == x.size
    Y = Y.cpu().numpy()
    yy = (Y.imag * Y.imag).astype(np.float32)
    sq = (Y.real.astype(np.float64) ** 2 + yy.astype(np.float64)).astype(np.float32).reshape(frames, N)
    ulps = np.abs(sq.view(np.int32).astype(np.int64) - P[False].view(np.int32).astype(np.int64))
    assert int(ulps.max()) <= 1, int(ulps.max())
    print(f"N {N}: largest FFT error / bound {float(np.max(ratio)):.3g}; {int(np.count_nonzero(ulps))} of "
          f"{ulps.size} values 1 ulp off the host's double-rounded fma")


@pytest.mark.gpu
def test_fused_spectrum_refusals():
    import torch
    from futuresdr_b200 import _lib
    from futuresdr_b200.blocks import SpectrumPipe
    from futuresdr_b200.context import default_context
    ctx = default_context().handle
    for n in (0, 16, 48, 1000, 16384, 1 << 20):
        with pytest.raises(_lib.B200SdrError):
            SpectrumPipe(n, 0.1, 1)
    h = ctypes.c_void_p()
    for decay in (-1e-7, -1.0, 1.0000001, 2.0, float("nan"), float("inf")):
        assert _lib.lib.b2s_spectrum_plan(ctx, 256, 1, decay, 1, 0.0, ctypes.byref(h)) == -1
        with pytest.raises(AssertionError):
            SpectrumPipe(256, decay, 1)
    assert _lib.lib.b2s_spectrum_plan(ctx, 256, 1, 0.1, 0, 0.0, ctypes.byref(h)) == -1
    with pytest.raises(_lib.B200SdrError):
        SpectrumPipe(256, 0.1, 0)
    blk = SpectrumPipe(256, 0.1, 1)
    x = torch.zeros(256 * 9, dtype=torch.complex64, device="cuda")
    o = torch.zeros(256 * 9 + 4, dtype=torch.float32, device="cuda")
    with pytest.raises(_lib.B200SdrError):
        blk.process(x[1:], o)                             # 8-byte offset
    for off in (1, 2, 3):
        with pytest.raises(_lib.B200SdrError):
            blk.process(x, o[off:])
    assert blk.process(x, o[4:]) == (256 * 9, 256 * 9)    # 16-byte aligned slices are accepted
