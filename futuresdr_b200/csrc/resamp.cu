// resamp.cu -- rational polyphase resampler (futuredsp::PolyphaseResamplingFir,
// crates/futuredsp/src/polyphase_resampling_fir.rs:70-124) on the device.
//
//   o[k] = sum_{t<T} i[floor(k*M/L) + t] * taps[L*(T-1-t) + (k*M mod L)],   T = ntaps / L
//
// Plans whose per-phase tap tables stay small (small L*M, resamp_slide_supported) run on the sliding-window kernel
// of the direct FIR (fir_direct.cu), the resampler being L decimate-by-M FIRs over one staged tile.  All others run
// resamp_kernel below: the host rearranges the taps once into bank-major, time-reversed rows  G[b][t] =
// taps[L*(T-1-t) + b]  (row pitch odd so lanes on different banks hit different smem banks).
// A CTA produces TK consecutive outputs: it stages the contiguous input span those outputs
// touch plus the bank table in shared memory, then each thread walks its outputs' T taps.  Plans whose span does not
// fit that tile (200 KiB) run resamp_naive_kernel, one thread per output reading global memory, so every plan that
// b2s_resamp_plan accepts executes.
// The (consumed, produced, status) triple follows :92-106 exactly (produced is a multiple of L).
#include "fir.cuh"

struct b2s_resamp {
    b2s_ctx *ctx = nullptr;
    b2s_kind kind = B2S_C32_F32;
    size_t ntaps = 0, interp = 1, decim = 1, T = 0;
    int pitch = 0;
    Buf<float> d_banks;          // [L][pitch]
    Buf<float> d_gtab;           // [L][M][Upad] per-phase taps of the sliding-window kernel (fir_direct.cu), or empty
};

namespace {

constexpr int kRsThreads = 256;
constexpr int kRsR = 4;          // outputs per thread that share one polyphase bank (tap reuse)

// A CTA produces R*S consecutive outputs, S = L*G >= 256 a multiple of L.  Thread slot tt < S owns
// the R outputs  k = kb + tt + r*S:  they share the bank (k*M mod L) and their input windows are
// exactly G*M items apart, so every tap fetched from shared memory feeds R MACs.
template <typename S, bool TAPS_IN_SMEM>
__global__ void __launch_bounds__(kRsThreads)
resamp_kernel(const S *__restrict__ in, S *__restrict__ out, const float *__restrict__ banks, int L, int M,
              int T, int pitch, long long n_out, int G, int span_max) {
    extern __shared__ __align__(16) unsigned char rsm[];
    S *xs = reinterpret_cast<S *>(rsm);
    float *gs = reinterpret_cast<float *>(rsm + (size_t)span_max * sizeof(S));
    const int Sg = L * G;                                       // outputs per r-slab
    const long long kb = (long long)blockIdx.x * kRsR * Sg;
    const long long klast = min(kb + (long long)kRsR * Sg, n_out) - 1;
    const long long base = kb * M / L;                          // first input item of the tile (kb*M/L exact: kb % L == 0)
    const int span = (int)(klast * M / L - base) + T;           // items the tile touches (<= span_max)
    for (int j = threadIdx.x; j < span; j += kRsThreads) xs[j] = in[base + j];
    if (TAPS_IN_SMEM)
        for (int j = threadIdx.x; j < L * pitch; j += kRsThreads) gs[j] = banks[j];
    __syncthreads();
    const float *g = TAPS_IN_SMEM ? gs : banks;
    const int step = G * M;                                     // input distance between a thread's outputs
    for (int tt = threadIdx.x; tt < Sg; tt += kRsThreads) {
        const long long k0 = kb + tt;
        if (k0 > klast) break;
        const long long km = (long long)tt * M;                 // (k0 - kb)*M ; kb*M is a multiple of L
        const int bank = (int)(km % L);
        const int i0 = (int)(km / L);
        const float *gb = g + bank * pitch;
        S acc[kRsR];
#pragma unroll
        for (int r = 0; r < kRsR; r++) acc[r] = zero_of<S>();
        int nr = kRsR;                                          // outputs of this thread inside n_out
        while (nr > 1 && k0 + (long long)(nr - 1) * Sg > klast) nr--;
        if (nr == kRsR) {
            for (int t = 0; t < T; t++) {
                const float tap = gb[t];
#pragma unroll
                for (int r = 0; r < kRsR; r++) mac(acc[r], xs[i0 + r * step + t], tap);
            }
        } else {
            for (int t = 0; t < T; t++) {
                const float tap = gb[t];
#pragma unroll
                for (int r = 0; r < kRsR; r++)
                    if (r < nr) mac(acc[r], xs[i0 + r * step + t], tap);
            }
        }
#pragma unroll
        for (int r = 0; r < kRsR; r++)
            if (r < nr) out[k0 + (long long)r * Sg] = acc[r];
    }
}

// Plans whose input span does not fit resamp_kernel's tile (large M/L, e.g. 1/100 or 4/125): one thread per output
// straight from global memory (L1/L2 cached), the same tap order as resamp_kernel.
template <typename S>
__global__ void resamp_naive_kernel(const S *__restrict__ in, S *__restrict__ out, const float *__restrict__ banks,
                                    int L, int M, int T, int pitch, long long n_out) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_out) return;
    const long long km = k * M;
    const S *x = in + km / L;
    const float *g = banks + (km % L) * pitch;
    S acc = zero_of<S>();
    for (int t = 0; t < T; t++) mac(acc, x[t], g[t]);
    out[k] = acc;
}

}  // namespace

extern "C" {

int32_t b2s_resamp_plan(b2s_ctx *ctx, b2s_kind kind, const float *taps, size_t ntaps, size_t interp,
                        size_t decim, b2s_resamp **out) {
    if (!ctx || !out || !taps) return b2s_fail(ctx, B2S_EINVAL, "b2s_resamp_plan: NULL argument");
    *out = nullptr;
    if (kind != B2S_F32_F32 && kind != B2S_C32_F32)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_resamp_plan: only f32xf32 and c32xf32 exist (polyphase_resampling_fir.rs:126-167)");
    if (interp == 0 || decim == 0 || ntaps == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_resamp_plan: zero interp/decim/ntaps");
    if (ntaps % interp != 0)   // assert!(taps.num_taps().is_multiple_of(interp))  (:56)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_resamp_plan: ntaps (%zu) must be a multiple of interp (%zu)", ntaps, interp);
    if (interp > 4096 || decim > 65536 || ntaps > (1u << 20)) return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_resamp_plan: factors too large");
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_resamp> r(new b2s_resamp());
    r->ctx = ctx; r->kind = kind; r->ntaps = ntaps; r->interp = interp; r->decim = decim; r->T = ntaps / interp;
    r->pitch = (int)(r->T | 1);                                   // odd row pitch
    std::vector<float> h(interp * r->pitch, 0.0f);
    for (size_t b = 0; b < interp; b++)
        for (size_t t = 0; t < r->T; t++) h[b * r->pitch + t] = taps[interp * (r->T - 1 - t) + b];   // :114
    B2S_TRY(r->d_banks.upload(ctx, h.data(), h.size(), "resampler taps"));
    std::vector<float> gt;
    if (resamp_slide_supported(interp, decim, r->T, kind_in_bytes(kind))) {
        gt = slide_table(taps, 1, interp, decim, r->T, 0);
        B2S_TRY(r->d_gtab.upload(ctx, gt.data(), gt.size(), "resampler phase taps"));
    }
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *out = r.release();
    return B2S_OK;
}

void b2s_resamp_destroy(b2s_resamp *r) { PlanDeleter<b2s_resamp>()(r); }

size_t b2s_resamp_length(const b2s_resamp *r) { return r ? r->ntaps : 0; }   // Filter::length = taps.num_taps() (:141-143)

int32_t b2s_resamp_exec(b2s_resamp *r, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                        size_t *consumed, size_t *produced, int32_t *status) {
    if (!r || !consumed || !produced || !status) return b2s_fail(r ? r->ctx : nullptr, B2S_EINVAL, "b2s_resamp_exec: NULL argument");
    b2s_ctx *ctx = r->ctx;
    const size_t L = r->interp, M = r->decim, T = r->T;
    // polyphase_resampling_fir.rs:92-106
    size_t p = sat_sub(sat_sub(n_in + 1, T) * L, 1) / M;
    p = (p / L) * L;
    if (p > n_out_cap) { p = (n_out_cap / L) * L; *status = B2S_INSUFFICIENT_OUTPUT; }
    else if (p == n_out_cap) *status = B2S_BOTH_SUFFICIENT;
    else *status = B2S_INSUFFICIENT_INPUT;
    *produced = p; *consumed = (p / L) * M;
    if (p == 0) return B2S_OK;
    if (!d_in || !d_out) return b2s_fail(ctx, B2S_EINVAL, "b2s_resamp_exec: NULL buffer");
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_resamp_exec");
    if (r->d_gtab)   // small L*M: L decimate-by-M sliding-window passes over one staged tile (fir_direct.cu)
        return resamp_slide_launch(ctx, r->kind, r->d_gtab.get(), L, M, T, d_in, n_in, d_out, p, ctx->stream);
    const size_t isz = kind_in_bytes(r->kind);
    const int G = (int)ceil_div((size_t)kRsThreads, L);                      // S = L*G >= 256 outputs per slab
    const size_t tile_out = (size_t)kRsR * L * G;
    const int span_max = (int)((tile_out * M) / L + T + 2);
    const size_t taps_bytes = L * r->pitch * sizeof(float);
    const size_t xs_bytes = round_up((size_t)span_max * isz, 16);
    const bool taps_smem = xs_bytes + taps_bytes <= 160 * 1024;
    const size_t smem = xs_bytes + (taps_smem ? taps_bytes : 0);
    if (xs_bytes > 200 * 1024) {   // the span does not fit one tile in shared memory
        const unsigned nb = (unsigned)ceil_div(p, (size_t)kRsThreads);
        if (r->kind == B2S_F32_F32)
            resamp_naive_kernel<float><<<nb, kRsThreads, 0, ctx->stream>>>((const float *)d_in, (float *)d_out, r->d_banks.get(),
                                                                           (int)L, (int)M, (int)T, r->pitch, (long long)p);
        else
            resamp_naive_kernel<float2><<<nb, kRsThreads, 0, ctx->stream>>>((const float2 *)d_in, (float2 *)d_out, r->d_banks.get(),
                                                                             (int)L, (int)M, (int)T, r->pitch, (long long)p);
        B2S_CHECK_LAUNCH(ctx);
        return B2S_OK;
    }
    const unsigned grid = (unsigned)ceil_div(p, tile_out);
#define RS_LAUNCH(S, TS)                                                                                     \
    do {                                                                                                     \
        constexpr auto kern = resamp_kernel<S, TS>;                                                          \
        if (smem > 48 * 1024) B2S_TRY(smem_optin<kern>(ctx, 216 * 1024));   /* the tile ceiling, not this plan's size */ \
        kern<<<grid, kRsThreads, smem, ctx->stream>>>((const S *)d_in, (S *)d_out, r->d_banks.get(), (int)L, (int)M, \
                                                      (int)T, r->pitch, (long long)p, G, (int)(xs_bytes / isz)); \
    } while (0)
    if (r->kind == B2S_F32_F32) { if (taps_smem) RS_LAUNCH(float, true); else RS_LAUNCH(float, false); }
    else { if (taps_smem) RS_LAUNCH(float2, true); else RS_LAUNCH(float2, false); }
#undef RS_LAUNCH
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

}  // extern "C"
