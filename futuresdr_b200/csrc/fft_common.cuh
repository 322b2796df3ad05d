// fft_common.cuh -- the shared-memory Stockham FFT core of every transform in the library (fft.cu, fir_fft.cu,
// spectrum.cu, chan.cu, synth.cu): in-register radix-2/4/8/16 forward DFTs, the padded shared-memory index, the
// batched CTA layout, the pass driver and the host-side twiddle table and size dispatch.
#pragma once
#include <cuda_runtime.h>

#include <cmath>
#include <type_traits>
#include <vector>

#include "common.cuh"

// The FFT plan (fft.cu), complete here so that other plans can own one as a sub-plan (PlanPtr<b2s_fft>).
struct b2s_fft {
    b2s_ctx *ctx = nullptr;
    size_t n = 0;
    int log2n = 0;
    int inverse = 0, shift = 0, has_norm = 0;
    float norm = 1.0f;
    Buf<float2> d_tw;           // W_N[k] = exp(-2 pi i k / N), k in [0, N)  (W_M for Bluestein)
    // Bluestein (chirp-z) path for lengths that are not a power of two
    bool bluestein = false;
    int log2m = 0;              // M = 2^log2m >= 2n - 1
    Buf<float2> d_chirp;        // w[k] = exp(-i pi k^2 / n), k in [0, n)
    Buf<float2> d_bhat;         // FFT_M of the wrapped conjugate chirp, pre-divided by M
    // LARGE transforms (n > 16384, or Bluestein with M > 16384): four-step through HBM on top of two shared-memory plans
    bool big = false;
    size_t big_m = 0, big_n1 = 0, big_n2 = 0;     // M = n1 * n2 (M = n for powers of two)
    PlanPtr<b2s_fft> sub1, sub2;                  // forward n1- and n2-point plans (no shift, no scale)
    Buf<float2> d_work;                           // 2 * M (four-step scratch) [+ 2 * M for Bluestein]
};

namespace fftk {

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ float2 mul_mi(float2 a) { return make_float2(a.y, -a.x); }   // a * (-i)

// ---- in-register forward DFTs, natural-order output ------------------------------------------
template <int R> struct Dft;
template <> struct Dft<2> {
    __device__ static __forceinline__ void run(float2 (&v)[2]) {
        const float2 a = v[0], b = v[1];
        v[0] = cadd(a, b); v[1] = csub(a, b);
    }
};
template <> struct Dft<4> {
    __device__ static __forceinline__ void run(float2 (&v)[4]) {
        const float2 t0 = cadd(v[0], v[2]), t1 = csub(v[0], v[2]);
        const float2 t2 = cadd(v[1], v[3]), t3 = mul_mi(csub(v[1], v[3]));
        v[0] = cadd(t0, t2); v[1] = cadd(t1, t3); v[2] = csub(t0, t2); v[3] = csub(t1, t3);
    }
};
template <> struct Dft<8> {
    __device__ static __forceinline__ void run(float2 (&v)[8]) {
        float2 e[4] = {v[0], v[2], v[4], v[6]}, o[4] = {v[1], v[3], v[5], v[7]};
        Dft<4>::run(e); Dft<4>::run(o);
        constexpr float h = 0.70710678118654752440f;
        o[1] = make_float2(h * (o[1].x + o[1].y), h * (o[1].y - o[1].x));      // * W8^1 = (1-i)/sqrt2
        o[2] = mul_mi(o[2]);                                                   // * W8^2 = -i
        o[3] = make_float2(h * (o[3].y - o[3].x), -h * (o[3].x + o[3].y));     // * W8^3 = (-1-i)/sqrt2
#pragma unroll
        for (int k = 0; k < 4; k++) { v[k] = cadd(e[k], o[k]); v[k + 4] = csub(e[k], o[k]); }
    }
};
template <> struct Dft<16> {
    __device__ static __forceinline__ void run(float2 (&v)[16]) {
        float2 e[8], o[8];
#pragma unroll
        for (int k = 0; k < 8; k++) { e[k] = v[2 * k]; o[k] = v[2 * k + 1]; }
        Dft<8>::run(e); Dft<8>::run(o);
        // W16^k = exp(-2 pi i k / 16)
        constexpr float c1 = 0.92387953251128675613f, s1 = 0.38268343236508977173f;
        constexpr float h = 0.70710678118654752440f;
        o[1] = cmul(o[1], make_float2(c1, -s1));
        o[2] = make_float2(h * (o[2].x + o[2].y), h * (o[2].y - o[2].x));
        o[3] = cmul(o[3], make_float2(s1, -c1));
        o[4] = mul_mi(o[4]);
        o[5] = cmul(o[5], make_float2(-s1, -c1));
        o[6] = make_float2(h * (o[6].y - o[6].x), -h * (o[6].x + o[6].y));
        o[7] = cmul(o[7], make_float2(-c1, -s1));
#pragma unroll
        for (int k = 0; k < 8; k++) { v[k] = cadd(e[k], o[k]); v[k + 8] = csub(e[k], o[k]); }
    }
};

__device__ __forceinline__ int pad(int i) { return i + (i >> 4); }

// Batched layout of 2^log2n-point transforms in a CTA of `cta_threads` threads: t threads per transform (one radix-16
// butterfly each, at most the whole CTA), fpb transforms per CTA, each in a padded row of np = n + n/16 elements.
// Kernels and their launchers both take it from here, so the shared-memory size always matches the kernel.
struct FftGeom {
    int n, t, fpb, np;
};
constexpr FftGeom fft_geom(int log2n, int cta_threads) {
    const int n = 1 << log2n;
    const int t = n / 16 < 1 ? 1 : (n / 16 > cta_threads ? cta_threads : n / 16);
    return FftGeom{n, t, cta_threads / t, n + n / 16};
}

// W_n[k] = exp(-2 pi i k / n), k in [0, n), evaluated in f64 and rounded to f32
inline std::vector<float2> twiddle_table(size_t n) {
    const double PI = 3.14159265358979323846264338327950288;
    std::vector<float2> tw(n);
    for (size_t k = 0; k < n; k++) {
        const double ang = -2.0 * PI * (double)k / (double)n;
        tw[k] = make_float2((float)std::cos(ang), (float)std::sin(ang));
    }
    return tw;
}

// f(std::integral_constant<int, L>{}) for L = log2n if LO <= log2n <= HI, else `otherwise`: one switch over the sizes a
// kernel template is instantiated for.
template <int LO, int HI, typename F>
int with_log2n(int log2n, int otherwise, F &&f) {
    if constexpr (LO > HI) return otherwise;
    else return log2n == LO ? f(std::integral_constant<int, LO>{}) : with_log2n<LO + 1, HI>(log2n, otherwise, f);
}


// v[r] *= w^r for r = 1..R-1, powers built by a log-depth product tree from ONE table load
// (15 dependent-free complex multiplies instead of 15 scattered 8-byte loads per butterfly: the
// table loads of a radix-16 pass cost ~16 L1 wavefronts each and made the FFT LSU-bound).
// Rounding: every power is at most 4 multiplies deep -> |error| <= ~4 ulp of the twiddle.
template <int R>
__device__ __forceinline__ void apply_twiddles(float2 (&v)[R], float2 w1) {
    if constexpr (R >= 2) v[1] = cmul(v[1], w1);
    if constexpr (R >= 4) {
        const float2 w2 = cmul(w1, w1), w3 = cmul(w2, w1);
        v[2] = cmul(v[2], w2); v[3] = cmul(v[3], w3);
        if constexpr (R >= 8) {
            const float2 w4 = cmul(w2, w2), w5 = cmul(w4, w1), w6 = cmul(w4, w2), w7 = cmul(w4, w3);
            v[4] = cmul(v[4], w4); v[5] = cmul(v[5], w5); v[6] = cmul(v[6], w6); v[7] = cmul(v[7], w7);
            if constexpr (R >= 16) {
                const float2 w8 = cmul(w4, w4);
                v[8] = cmul(v[8], w8); v[9] = cmul(v[9], cmul(w8, w1)); v[10] = cmul(v[10], cmul(w8, w2));
                v[11] = cmul(v[11], cmul(w8, w3)); v[12] = cmul(v[12], cmul(w8, w4)); v[13] = cmul(v[13], cmul(w8, w5));
                v[14] = cmul(v[14], cmul(w8, w6)); v[15] = cmul(v[15], cmul(w8, w7));
            }
        }
    }
}

template <int LOG2N> struct Plan;   // radices per pass
template <> struct Plan<1>  { static constexpr int P = 1, R0 = 2,  R1 = 1,  R2 = 1, R3 = 1; };
template <> struct Plan<2>  { static constexpr int P = 1, R0 = 4,  R1 = 1,  R2 = 1, R3 = 1; };
template <> struct Plan<3>  { static constexpr int P = 1, R0 = 8,  R1 = 1,  R2 = 1, R3 = 1; };
template <> struct Plan<4>  { static constexpr int P = 1, R0 = 16, R1 = 1,  R2 = 1, R3 = 1; };
template <> struct Plan<5>  { static constexpr int P = 2, R0 = 8,  R1 = 4,  R2 = 1, R3 = 1; };
template <> struct Plan<6>  { static constexpr int P = 2, R0 = 8,  R1 = 8,  R2 = 1, R3 = 1; };
template <> struct Plan<7>  { static constexpr int P = 2, R0 = 16, R1 = 8,  R2 = 1, R3 = 1; };
template <> struct Plan<8>  { static constexpr int P = 2, R0 = 16, R1 = 16, R2 = 1, R3 = 1; };
template <> struct Plan<9>  { static constexpr int P = 3, R0 = 8,  R1 = 8,  R2 = 8, R3 = 1; };
template <> struct Plan<10> { static constexpr int P = 3, R0 = 16, R1 = 8,  R2 = 8, R3 = 1; };
template <> struct Plan<11> { static constexpr int P = 3, R0 = 16, R1 = 16, R2 = 8, R3 = 1; };
template <> struct Plan<12> { static constexpr int P = 3, R0 = 16, R1 = 16, R2 = 16, R3 = 1; };
template <> struct Plan<13> { static constexpr int P = 4, R0 = 16, R1 = 8,  R2 = 8, R3 = 8; };
template <> struct Plan<14> { static constexpr int P = 4, R0 = 16, R1 = 16, R2 = 8, R3 = 8; };


template <int LOG2N> constexpr int plan_radix(int p) {        // radix of pass p
    using PL = Plan<LOG2N>;
    return p == 0 ? PL::R0 : p == 1 ? PL::R1 : p == 2 ? PL::R2 : PL::R3;
}
template <int LOG2N> constexpr int plan_ns(int p) {           // sub-transform size before pass p
    return p == 0 ? 1 : plan_ns<LOG2N>(p - 1) * plan_radix<LOG2N>(p - 1);
}

// The base twiddle of butterfly j of a pass: loaded from the table after the pass's barrier (TwTable), or held in
// registers from a fetch before the PREVIOUS pass ran (TwAhead) -- with a fixed number of butterflies per thread the
// index depends on the thread alone, so the load is in flight across the barrier instead of being waited for right
// after it.  The held values cost registers, which is why the choice is per kernel (Tw below).
struct TwTable {
    const float2 *__restrict__ tw;
    template <int N, int R, int NS> __device__ __forceinline__ float2 get(int j, int) const {
        return __ldg(tw + (j & (NS - 1)) * (N / (NS * R)));
    }
};
template <int N, int R, int NS, int T> struct TwAhead {
    static constexpr int ITER = (N / R) / T > 0 ? (N / R) / T : 1;
    float2 w[ITER];
    __device__ __forceinline__ void fetch(const float2 *__restrict__ tw, int t) {
#pragma unroll
        for (int it = 0; it < ITER; it++) w[it] = __ldg(tw + ((t + it * T) & (NS - 1)) * (N / (NS * R)));
    }
    template <int N_, int R_, int NS_> __device__ __forceinline__ float2 get(int, int it) const { return w[it]; }
};

// Where passes 1.. of fft_passes take their base twiddles from: Table = TwTable, Ahead = TwAhead.
enum class Tw { Table, Ahead };

// One Stockham pass: loads through `load`, optional CTA barrier (in-place passes), twiddles, DFT,
// stores through `store`, optional CTA barrier.
template <int N, int R, int NS, int T, typename LoadF, typename StoreF, typename TwF>
__device__ __forceinline__ void ss_pass_tw(LoadF load, StoreF store, TwF twf, int t, bool sync_between,
                                           bool sync_after = true) {
    constexpr int NB = N / R, ITER = NB / T;
    static_assert(NB % T == 0, "butterflies must tile the threads");
    float2 v[ITER][R];
#pragma unroll
    for (int it = 0; it < ITER; it++) {
        const int j = t + it * T;
#pragma unroll
        for (int r = 0; r < R; r++) v[it][r] = load(j + r * NB);
    }
    if (sync_between) __syncthreads();
#pragma unroll
    for (int it = 0; it < ITER; it++) {
        const int j = t + it * T;
        if constexpr (NS > 1) apply_twiddles<R>(v[it], twf.template get<N, R, NS>(j, it));
        Dft<R>::run(v[it]);
        const int j0 = (j / NS) * NS * R + (j & (NS - 1));
#pragma unroll
        for (int r = 0; r < R; r++) store(j0 + r * NS, v[it][r]);
    }
    if (sync_after) __syncthreads();
}

template <Tw TW, int LOG2N, int P, int T>
__device__ __forceinline__ auto pass_twiddles(const float2 *__restrict__ tw, int t) {
    if constexpr (TW == Tw::Ahead) {
        TwAhead<1 << LOG2N, plan_radix<LOG2N>(P), plan_ns<LOG2N>(P), T> w;
        w.fetch(tw, t);
        return w;
    } else {
        return TwTable{tw};
    }
}

// Passes P.. of the plan, in place in `sm` except the last, which writes through `last_store`; `w` holds pass P's
// base twiddles.  With Tw::Ahead the next pass's twiddles are fetched before this pass runs.
template <int LOG2N, int T, Tw TW, int P, typename StoreF, typename TwF>
__device__ __forceinline__ void fft_passes_from(StoreF last_store, float2 *sm, const float2 *__restrict__ tw, int t,
                                                bool sync_last, const TwF &w) {
    constexpr int N = 1 << LOG2N, R = plan_radix<LOG2N>(P), NS = plan_ns<LOG2N>(P);
    auto ld_sm = [&](int idx) { return sm[pad(idx)]; };
    if constexpr (P + 1 == Plan<LOG2N>::P) {
        ss_pass_tw<N, R, NS, T>(ld_sm, last_store, w, t, sync_last, sync_last);
    } else {
        const auto wn = pass_twiddles<TW, LOG2N, P + 1, T>(tw, t);
        ss_pass_tw<N, R, NS, T>(ld_sm, [&](int idx, float2 v) { sm[pad(idx)] = v; }, w, t, true);
        fft_passes_from<LOG2N, T, TW, P + 1>(last_store, sm, tw, t, sync_last, wn);
    }
}

struct NoHook {
    __device__ __forceinline__ void operator()() const {}
};

// Runs a whole LOG2N-point forward FFT as Stockham passes through the padded smem buffer `sm`.
// Pass 0 reads through `first_load(idx)`, the last pass writes through `last_store(idx, v)`, the
// passes in between read and write `sm`.  first_reads_smem: pass 0's source is `sm` itself.
// sync_last = false drops the barriers of the last pass (between its loads and stores, and after it) -- for a last
// store that leaves shared memory at the end of the kernel.
// `after_first` runs right after pass 0: from then on pass 0's source is free (spectrum.cu starts the asynchronous
// fetch of the next transform's input there).  TW: where passes 1.. take their base twiddles (see TwTable).
template <int LOG2N, int T, Tw TW, typename LoadF, typename StoreF, typename HookF = NoHook>
__device__ __forceinline__ void fft_passes(LoadF first_load, StoreF last_store, float2 *sm,
                                           const float2 *__restrict__ tw, int t, bool first_reads_smem,
                                           bool sync_last = true, HookF after_first = {}) {
    constexpr int N = 1 << LOG2N, R0 = Plan<LOG2N>::R0;
    if constexpr (Plan<LOG2N>::P == 1) {
        ss_pass_tw<N, R0, 1, T>(first_load, last_store, TwTable{tw}, t, first_reads_smem, sync_last);
        after_first();
    } else {
        const auto w1 = pass_twiddles<TW, LOG2N, 1, T>(tw, t);
        ss_pass_tw<N, R0, 1, T>(first_load, [&](int idx, float2 v) { sm[pad(idx)] = v; }, TwTable{tw}, t,
                                first_reads_smem);
        after_first();
        fft_passes_from<LOG2N, T, TW, 1>(last_store, sm, tw, t, sync_last, w1);
    }
}

}  // namespace fftk
