// spectrum.cu -- the spectrum pipe  Fft(N, Forward, shift) -> Apply(|x|^2) -> MovingAvg<N>(decay, history)
// [-> k*log10]  fused into ONE pass over the samples (SURVEY.md 8f-3; examples/spectrum/src/bin/cpu.rs:21-28,
// src/blocks/fft.rs:160-221, src/blocks/moving_avg.rs:78-116; the reference's own GPU prior art fuses
// reduce + shift + log10 the same way, perf/burn/src/bin/fft-cubecl-kernel.rs:115-146).
//
// Only  8 B/sample in  and  4/history B/sample out  touch HBM (the unfused chain moves 32 B/sample).  The obstacle is
// the moving average: per bin it is a recurrence over ALL frames of the stream,
//     avg <- (1-d)*avg + d*t      (t finite; avg <- (1-d)*avg otherwise)            moving_avg.rs:85-90
// which is linear in (avg, t), so it is evaluated as a two-level scan:
//   1. spectrum_kernel : a thread group owns C consecutive frames; per frame it runs the N-point Stockham FFT in
//      shared memory (fft_common.cuh), takes |X|^2, and advances a LOCAL average (zero start state, registers, the
//      reference's un-fused multiply/add order); every history-th frame of the STREAM it stores the local average,
//      and at the end the group's final local state.
//   2. spectrum_scan   : per bin, carry_{g+1} = final_g + a^{C_g} * carry_g  across the groups (a = 1-d; carry_0 is
//      the state left by the previous call) -- a warp per bin composes the affine maps with a shuffle scan.
//   3. spectrum_fixup  : emitted[o] += a^k * carry_g  (k = frames of group g up to and including the emitting one),
//      then the optional k*log10.
// In real arithmetic this IS the reference's recurrence; in f32 the rounding order of the carried-in term differs,
// so parity with the oracle is a bound per emitted value of every bin, not bit equality: within 2 B + 4 u V of the
// float64 recurrence V, B the rounding-error bound of the sequential f32 recurrence (tests/test_gpu_spectrum_bins.py)
// -- the unfused bit-exact blocks (fft.cu, apply.cu, mavg.cu) remain.  The weights a^k, a^C, the scan's states and
// the fix-up's product are float64: a^k leaves f32's normal range long before a^k * carry does (k > 38 at decay 0.9,
// k > 149 at decay 0.5), and an f32 weight would lose the carried-in term there.  Why not one exact pass: a bin's chain
// is 2 dependent f32 operations per frame (~8 cycles), i.e. at most ~240 M frames/s per bin however many SMs there
// are.
#include <cmath>

#include "common.cuh"
#include "fft_common.cuh"

struct b2s_spectrum {
    b2s_ctx *ctx = nullptr;
    size_t n = 0;
    int log2n = 0, shift = 0;
    size_t history = 1;
    float decay = 0.1f, log10_k = 0.0f;
    Buf<float2> d_tw;
    Buf<float> d_avg;              // [n] running average, OUTPUT (post-shift) bin order
    Buf<float> d_final;            // [groups][n] local final states / carries (grown on demand)
    Buf<double> d_pow;             // a^k, k = 0..cap (float64: see the top of the file)
    size_t i = 0;                  // frames since the last emission (moving_avg.rs: self.i)
    int resident = 0;              // CTAs per SM of the kernel instantiation (occupancy query, first exec)
};

namespace {
using namespace fftk;
constexpr int kSpThreads = 256;

struct SpArgs {
    const float2 *in;
    float *out;                // [n_emit][N]
    float *fin;                // [groups][N]
    const float2 *tw;
    long long nframes, C;      // frames in this call, frames per group
    int groups, shift, history, i0;
    float a, d;
};

// The next frame of a group is fetched with cp.async into a raw staging row while the current one is being
// transformed: the first FFT pass reads the staging row, and from the barrier that ends it the row is free again, so
// the fetch of frame c+1 overlaps passes 2.. and the averaging of frame c.  (The first version read the frame with
// plain loads at the top of every round, which serialized the load and compute phases.)
template <int LOG2N>
__global__ void __launch_bounds__(kSpThreads, (LOG2N <= 12 ? 3 : 1)) spectrum_kernel(const SpArgs p) {
    constexpr FftGeom G = fft_geom(LOG2N, kSpThreads);
    constexpr int N = G.n, T = G.t, FPB = G.fpb;
    constexpr int NB = N / T;                                                            // bins per thread
    extern __shared__ __align__(16) unsigned char ssm[];
    const int t = threadIdx.x % T, fl = threadIdx.x / T;
    const int g = blockIdx.x * FPB + fl;
    const bool live = g < p.groups;
    float2 *sm = reinterpret_cast<float2 *>(ssm) + (size_t)fl * G.np;         // padded FFT buffer of this group
    float2 *raw = reinterpret_cast<float2 *>(ssm) + (size_t)FPB * G.np + (size_t)fl * N;   // staging row (next frame)
    float *sP = reinterpret_cast<float *>(sm);              // |X|^2 of the current frame (aliases the FFT buffer)
    const long long f0 = (long long)(live ? g : p.groups - 1) * p.C;
    const long long nf = live ? min(p.C, p.nframes - f0) : 0;
    float avg[NB];
#pragma unroll
    for (int k = 0; k < NB; k++) avg[k] = 0.0f;
    auto fetch = [&](long long c) {                          // frame c of this group -> raw (idle rounds re-fetch frame 0)
        const float4 *src = reinterpret_cast<const float4 *>(p.in + (f0 + (c < nf ? c : 0)) * N);
        for (int i = t; i < N / 2; i += T) cp_async::cg16(reinterpret_cast<float4 *>(raw) + i, src + i);
        cp_async::commit();
    };
    fetch(0);
    for (long long c = 0; c < p.C; c++) {                   // every group of the CTA runs C rounds (barriers inside)
        const bool act = c < nf;
        cp_async::wait<0>();
        __syncthreads();                                     // raw holds frame c; everyone is done with sP of frame c-1
        fft_passes<LOG2N, T, Tw::Ahead>([&](int idx) { return raw[idx]; },
                                        [&](int idx, float2 v) { sP[idx] = fmaf(v.x, v.x, v.y * v.y); },   // norm_sqr
                                        sm, p.tw, t, false, true, [&]() { if (c + 1 < p.C) fetch(c + 1); });
        if (act) {
            const long long fs = f0 + c;                     // frame index within the call
            const bool emit = ((p.i0 + fs + 1) % p.history) == 0;
            float *orow = p.out + ((p.i0 + fs + 1) / p.history - 1) * N;
#pragma unroll
            for (int k = 0; k < NB; k++) {
                const int b = t + k * T;
                const float tv = sP[b];
                const float dec = __fmul_rn(p.a, avg[k]);    // un-fused, reference order: (1-d)*avg + d*t
                avg[k] = isfinite(tv) ? __fadd_rn(dec, __fmul_rn(p.d, tv)) : dec;
                if (emit) orow[p.shift ? ((b + N / 2) & (N - 1)) : b] = avg[k];
            }
        }
    }
    if (live) {
#pragma unroll
        for (int k = 0; k < NB; k++) {
            const int b = t + k * T;
            p.fin[(size_t)g * N + (p.shift ? ((b + N / 2) & (N - 1)) : b)] = avg[k];
        }
    }
}

// Carry scan across the groups.  A CTA owns 32 adjacent bins (the lanes of a warp: every load / store below is one
// coalesced 128-byte line) and cuts the groups into 32 segments, one per warp:
//   1. each warp composes the affine maps  x -> final_g + A_g * x  of its segment (sequential over ~groups/32 groups);
//   2. the 32 composites of a bin are scanned through shared memory (sequential over segments, 32 lanes = 32 bins);
//   3. each warp walks its segment again with the now known incoming state and overwrites fin[g][bin] with the state
//      group g STARTS from; the state after the call goes to avg[].
// (History: a warp per bin with the lanes striding over groups -- 4-byte loads 8 KiB apart -- took 207 us for 7 MB of
// carries, as long as the FFT kernel itself; doing the row fix-up inside step 3 left ~200 dependent memory round trips
// per warp and took 224 us.  Carries and fix-up are separate again, each fully parallel.)
constexpr int kScanSegs = 32;
__global__ void __launch_bounds__(32 * kScanSegs)
spectrum_scan(float *fin, float *avg, int n, int groups, double A, double A_last) {
    __shared__ double sL[kScanSegs][33], sM[kScanSegs][33], sX[kScanSegs][33];
    const int lane = threadIdx.x & 31, seg = threadIdx.x >> 5;
    const int bin = blockIdx.x * 32 + lane;
    const bool live = bin < n;
    const int per = (groups + kScanSegs - 1) / kScanSegs;
    const int g0 = min(seg * per, groups), g1 = min(g0 + per, groups);
    double L = 0.0, M = 1.0;
    if (live) {
#pragma unroll 4
        for (int g = g0; g < g1; g++) {
            const double Ag = (g == groups - 1) ? A_last : A;
            L = fma(Ag, L, (double)fin[(size_t)g * n + bin]);
            M *= Ag;
        }
    }
    sL[seg][lane] = L; sM[seg][lane] = M;
    __syncthreads();
    if (seg == 0) {
        double x = live ? avg[bin] : 0.0;
        for (int sgm = 0; sgm < kScanSegs; sgm++) {
            sX[sgm][lane] = x;
            x = fma(sM[sgm][lane], x, sL[sgm][lane]);
        }
        if (live) avg[bin] = (float)x;                       // state after the call
    }
    __syncthreads();
    if (!live) return;
    double x = sX[seg][lane];
#pragma unroll 4
    for (int g = g0; g < g1; g++) {
        const double Ag = (g == groups - 1) ? A_last : A;
        const float f = fin[(size_t)g * n + bin];
        fin[(size_t)g * n + bin] = (float)x;                 // carry INTO group g
        x = fma(Ag, x, (double)f);
    }
}

// emitted[row] += a^k * carry_g  (k = frames of group g up to and including the emitting one), then the optional
// k*log10.  One row (or a 1024-bin slice of it) per CTA: the group / power look-up is per CTA, accesses are float4.
__global__ void __launch_bounds__(256)
spectrum_fixup(float *out, const float *__restrict__ carry, const double *__restrict__ apow, int n, long long C,
               int history, int i0, float log10_k) {
    const long long row = blockIdx.x;
    const long long f = (row + 1) * history - i0 - 1;          // frame (within the call) that emitted this row
    const long long g = f / C;
    const double w = apow[(int)(f - g * C) + 1];
    const int b = (blockIdx.y * 256 + threadIdx.x) * 4;
    if (b >= n) return;
    float4 v = *reinterpret_cast<float4 *>(out + row * n + b);
    const float4 c = *reinterpret_cast<const float4 *>(carry + (size_t)g * n + b);
    v.x = (float)fma(w, (double)c.x, (double)v.x); v.y = (float)fma(w, (double)c.y, (double)v.y);
    v.z = (float)fma(w, (double)c.z, (double)v.z); v.w = (float)fma(w, (double)c.w, (double)v.w);
    if (log10_k != 0.0f) { v.x = log10_k * log10f(v.x); v.y = log10_k * log10f(v.y); v.z = log10_k * log10f(v.z); v.w = log10_k * log10f(v.w); }
    *reinterpret_cast<float4 *>(out + row * n + b) = v;
}

constexpr size_t spectrum_smem(int log2n) {           // per transform slot: the padded FFT buffer and the staging row
    const FftGeom g = fft_geom(log2n, kSpThreads);
    return (size_t)g.fpb * (g.np + g.n) * sizeof(float2);
}

template <int LOG2N>
int32_t launch_spectrum(b2s_spectrum *p, const SpArgs &a, cudaStream_t stream) {
    constexpr size_t smem = spectrum_smem(LOG2N);
    B2S_TRY(smem_optin<spectrum_kernel<LOG2N>>(p->ctx, smem));
    const unsigned grid = (unsigned)ceil_div((size_t)a.groups, (size_t)fft_geom(LOG2N, kSpThreads).fpb);
    spectrum_kernel<LOG2N><<<grid, kSpThreads, smem, stream>>>(a);
    B2S_CHECK_LAUNCH(p->ctx);
    return B2S_OK;
}

}  // namespace

extern "C" {

int32_t b2s_spectrum_plan(b2s_ctx *ctx, size_t n, int32_t fft_shift, float decay_factor, size_t history_size,
                          float log10_scale, b2s_spectrum **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_spectrum_plan: NULL argument");
    *out = nullptr;
    if (n < 32 || (n & (n - 1)) || n > 8192)
        return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_spectrum_plan: n must be a power of two in [32, 8192] (got %zu)", n);
    // moving_avg.rs:62-65 asserts this
    if (!(decay_factor >= 0.0f && decay_factor <= 1.0f)) return b2s_fail(ctx, B2S_EINVAL, "decay_factor must be in [0, 1]");
    if (history_size == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_spectrum_plan: history_size must be > 0");
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_spectrum> p(new b2s_spectrum());
    p->ctx = ctx; p->n = n; p->shift = fft_shift != 0; p->decay = decay_factor; p->history = history_size;
    p->log10_k = log10_scale;
    while (((size_t)1 << p->log2n) < n) p->log2n++;
    const std::vector<float2> tw = twiddle_table(n);
    B2S_TRY(p->d_tw.upload(ctx, tw.data(), n, "spectrum twiddles"));
    B2S_TRY(p->d_avg.alloc(ctx, n, "spectrum average"));
    B2S_CUDA(ctx, cudaMemsetAsync(p->d_avg.get(), 0, n * sizeof(float), ctx->stream));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *out = p.release();
    return B2S_OK;
}

void b2s_spectrum_destroy(b2s_spectrum *p) { PlanDeleter<b2s_spectrum>()(p); }

int32_t b2s_spectrum_reset(b2s_spectrum *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "spectrum is NULL");
    DeviceGuard g(p->ctx->device);
    p->i = 0;
    B2S_CUDA(p->ctx, cudaMemsetAsync(p->d_avg.get(), 0, p->n * sizeof(float), p->ctx->stream));
    return B2S_OK;
}

// One call == Fft::work + Apply::work + MovingAvg::work on the same slices: frames = min(n_in / N, what fits the
// output: every history-th frame emits N floats, moving_avg.rs:82) ; consumed = frames * N input items,
// produced = emitted rows * N floats.
int32_t b2s_spectrum_exec(b2s_spectrum *p, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                          size_t *consumed, size_t *produced) {
    if (!p || !consumed || !produced) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_spectrum_exec: NULL argument");
    b2s_ctx *ctx = p->ctx;
    const size_t N = p->n, h = p->history;
    size_t frames = n_in / N;
    const size_t rows_cap = n_out_cap / N;
    // MovingAvg::work's loop condition (moving_avg.rs:82): a chunk is only taken while one more output row would
    // still fit, so the frame that fills the last row is the last one processed
    const size_t max_frames = rows_cap == 0 ? 0 : (h - p->i) + (rows_cap - 1) * h;
    if (frames > max_frames) frames = max_frames;
    const size_t rows = (p->i + frames) / h;
    *consumed = frames * N; *produced = rows * N;
    if (frames == 0) return B2S_OK;
    if (!d_in || (rows && !d_out)) return b2s_fail(ctx, B2S_EINVAL, "b2s_spectrum_exec: NULL buffer");
    if ((reinterpret_cast<uintptr_t>(d_in) & 15) || (rows && (reinterpret_cast<uintptr_t>(d_out) & 15)))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_spectrum_exec: the input and output slices must be 16-byte aligned");
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_spectrum_exec");
    cudaStream_t st = ctx->stream;
    // thread groups: one wave of resident CTAs when the call is long enough, never fewer than 4 frames per group
    const int FPB = fft_geom(p->log2n, kSpThreads).fpb;
    if (!p->resident)                                        // CTAs of this size's kernel that fit one SM
        B2S_TRY((with_log2n<5, 13>(p->log2n, B2S_OK, [&](auto L) {
            return smem_optin<spectrum_kernel<L>>(ctx, spectrum_smem(L), kSpThreads, &p->resident);
        })));
    const size_t resident = (size_t)std::max(1, p->resident);
    const size_t g_target = (size_t)ctx->sm_count * resident * FPB;
    const size_t C = std::max<size_t>(4, ceil_div(frames, g_target));
    const size_t groups = ceil_div(frames, C);
    if (p->d_final.size() < groups * N) B2S_TRY(p->d_final.reserve(ctx, groups * N * 5 / 4, "spectrum carries"));
    if (p->d_pow.size() < C + 1) {
        const size_t want = (C + 1) * 2;
        B2S_TRY(p->d_pow.reserve(ctx, want, "spectrum powers"));
        std::vector<double> pw(want);
        const double a = (double)(1.0f - p->decay);
        for (size_t k = 0; k < want; k++) pw[k] = std::pow(a, (double)k);
        B2S_CUDA(ctx, cudaMemcpyAsync(p->d_pow.get(), pw.data(), want * sizeof(double), cudaMemcpyHostToDevice, st));
        B2S_CUDA(ctx, cudaStreamSynchronize(st));            // pw is a stack-owned vector
    }
    SpArgs a;
    a.in = (const float2 *)d_in; a.out = (float *)d_out; a.fin = p->d_final.get(); a.tw = p->d_tw.get();
    a.nframes = (long long)frames; a.C = (long long)C; a.groups = (int)groups; a.shift = p->shift;
    a.history = (int)h; a.i0 = (int)p->i; a.a = 1.0f - p->decay; a.d = p->decay;
    const int32_t rc = with_log2n<5, 13>(p->log2n, B2S_EUNSUPPORTED, [&](auto L) { return launch_spectrum<L>(p, a, st); });
    if (rc != B2S_OK) return rc == B2S_EUNSUPPORTED ? b2s_fail(ctx, rc, "b2s_spectrum_exec: unsupported size") : rc;
    const double ad = (double)(1.0f - p->decay);
    const size_t c_last = frames - (groups - 1) * C;
    spectrum_scan<<<(unsigned)ceil_div(N, (size_t)32), 32 * kScanSegs, 0, st>>>(
        p->d_final.get(), p->d_avg.get(), (int)N, (int)groups, std::pow(ad, (double)C), std::pow(ad, (double)c_last));
    B2S_CHECK_LAUNCH(ctx);
    if (rows) {
        dim3 grid((unsigned)rows, (unsigned)ceil_div(N, (size_t)1024));
        spectrum_fixup<<<grid, 256, 0, st>>>((float *)d_out, p->d_final.get(), p->d_pow.get(), (int)N, (long long)C, (int)h, (int)p->i, p->log10_k);
        B2S_CHECK_LAUNCH(ctx);
    }
    p->i = (p->i + frames) % h;
    return B2S_OK;
}

}  // extern "C"
