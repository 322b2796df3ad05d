// synth.cu -- polyphase synthesizer (src/blocks/pfb/synthesizer.rs:52-144), the dual of chan.cu:
// SURVEY.md §8f row 2.
//
// Reference: per input vector v (one sample from each of the N input streams) an un-normalised
// N-point inverse FFT "spins" the vector, element w is pushed into window w, and once the windows
// are filled arm w (taps[w::N]) filters window w into the next output item -- N outputs per vector.
// Device form: (1) gather the channel-major inputs into vectors and run the batched inverse FFT of
// fft.cu; (2) one thread per (vector, arm) dots the T newest spun samples of its slot (history
// buffer + this call) with its arm and writes out[(v - v0) * N + w] -- coalesced in w.
// The windows are the shared window buffer of pfb_common.cuh (spun sample w of vector v is item v*N + w
// of its stream, so all windows move in lockstep); the loop condition of :95-97
// (`out.len() - produced > N || !all_windows_filled`) is evaluated in closed form.
#include <cstdlib>

#include "pfb_common.cuh"

struct b2s_synth {
    b2s_ctx *ctx = nullptr;
    size_t N = 0, T = 0;
    PfbBankTaps taps;               // arm w filters window w
    PfbWindows win;                 // N windows: spun sample w of every vector goes to window w
    PlanPtr<b2s_fft> ifft;
    Buf<float2> d_tmp;              // two halves: gathered vectors, spun vectors
};

namespace {

// outputs for steady vectors u in [u0, k2): u = -1 is the vector that completed the fill (history only)
__global__ void synth_bank_kernel(const float2 *__restrict__ spun /* steady vectors, u = 0 first */,
                                  const float2 *__restrict__ hist, const float *__restrict__ arms,
                                  float2 *__restrict__ out, int N, int T, int u0, long long k2) {
    const long long total = (k2 - u0) * N;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += stride) {
        const long long u = u0 + g / N;
        const int w = (int)(g % N);
        const float *a = arms + w;                                // tap-major table: arm w, tap j at a[j * N] (coalesced across w)
        float re = 0.f, im = 0.f;
        for (int j = T - 1; j >= 0; j--) {                       // oldest first, like the reference's t = 0..T-1
            const long long up = u - j;
            const float2 x = up >= 0 ? __ldg(spun + up * N + w) : hist[(size_t)w * T + (T + up)];
            const float tap = __ldg(a + (size_t)j * N);
            re = fmaf(x.x, tap, re); im = fmaf(x.y, tap, im);
        }
        out[g] = make_float2(re, im);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// FUSED steady state (N a power of two <= 256, T <= 32): gather + N-point inverse FFT + FIR bank in ONE kernel --
// 8 B/sample in, 8 B/sample out, the spun vectors never touch HBM (the three kernels above move 40 B/sample).  A CTA
// owns a contiguous range of tiles of OB = 4096/N vectors and keeps the last TPAD-1 spun vectors of the previous tile
// in a shared-memory ring (its first tile is preceded by a warm-up tile that only fills the ring):
//   A. the tile's OB vectors are read channel-major (OB consecutive items per input stream: coalesced) into a staging
//      array with an odd pitch;
//   B. every vector is spun by the Stockham passes of fft_common.cuh (inverse = conj o FFT o conj), the first pass
//      reading the staging array transposed, the last one writing row (TPAD-1+v) of the ring;
//   C. thread (arm w, run of RL vectors) streams column w of the ring through registers once -- each spun sample is
//      multiplied into every output of the run that contains it (taps in registers, oldest first like
//      synthesizer.rs:106-118) -- and stores out[u*N + w], coalesced in w;
//   D. the last TPAD-1 rows move to the top of the ring; the CTA that owns the last tile leaves the T newest spun
//      vectors in the plan's history buffer for the next call.
// The first vectors of a call (windows still reaching into the previous call's history; one tile, more when a tile is
// shorter than the history), the window fill and other bank shapes take the three-kernel path.
// ---------------------------------------------------------------------------------------------------------------
template <int LOG2N, int TPAD, bool PADDED>
__global__ void __launch_bounds__(256) synth_fused_kernel(const float2 *__restrict__ in, long long in_stride,
                                                          const float *__restrict__ arms_pad, const float2 *__restrict__ tw,
                                                          float2 *__restrict__ out, float2 *__restrict__ hist, int T,
                                                          long long k2, int ntiles, int tiles_per_cta) {
    using namespace fftk;
    constexpr FftGeom G = fft_geom(LOG2N, 256);
    constexpr int N = G.n, TT = G.t, NP = G.np;              // TT threads per transform
    constexpr int OB = G.fpb;                                // vectors per tile
    constexpr int RUNS = 256 / N, RL = OB / RUNS;
    constexpr int XP = OB + 1;                               // odd pitch of the gather staging
    constexpr int WARM = (TPAD - 1 + OB - 1) / OB;           // warm-up tiles that fill TPAD-1 rows of history (1 unless OB < TPAD-1)
    extern __shared__ __align__(16) unsigned char ysm[];
    float2 *Xs = reinterpret_cast<float2 *>(ysm);            // [N][XP]
    float2 *Vf = Xs + (size_t)N * XP;                        // [OB][NP]
    float2 *Sb = Vf + (size_t)OB * NP;                       // [TPAD-1+OB][N]  spun vectors, oldest row first
    const int tid = threadIdx.x;
    const int w = tid % N, run = tid / N;
    float tap[TPAD];
#pragma unroll
    for (int j = 0; j < TPAD; j++) tap[j] = __ldg(arms_pad + (size_t)j * N + w);

    const int t0 = blockIdx.x * tiles_per_cta, t1 = min(t0 + tiles_per_cta, ntiles);
    for (int t = t0 - WARM; t < t1; t++) {                   // t < t0: warm-up tiles (fill the ring, emit nothing)
        const long long v0 = (long long)OB * (t + WARM);     // tile t covers vectors [OB*(t+WARM), +OB); vectors < OB*WARM: generic path
        // ---- A: gather
        for (int e = tid; e < N * OB; e += 256) {
            const int ch = e / OB, v = e % OB;
            Xs[(size_t)ch * XP + v] = (v0 + v < k2) ? __ldg(in + (long long)ch * in_stride + v0 + v) : make_float2(0.f, 0.f);
        }
        __syncthreads();
        // ---- B: spin
        {
            const int ol = tid / TT, tt = tid % TT;
            float2 *sm = Vf + (size_t)ol * NP;
            fft_passes<LOG2N, TT, Tw::Ahead>([&](int idx) { const float2 x = Xs[(size_t)idx * XP + ol]; return make_float2(x.x, -x.y); },
                                             [&](int idx, float2 v) { Sb[(size_t)(TPAD - 1 + ol) * N + idx] = make_float2(v.x, -v.y); },
                                             sm, tw, tt, false);
        }
        // (fft_passes ends with a CTA barrier)
        if (t >= t0) {
            // ---- C: FIR bank
            float2 acc[RL];
            // ring row (run*RL + k) <-> vector v0 + run*RL + k - (TPAD-1)
            pfb_bank_column<N, RL, TPAD, PADDED>(Sb + (size_t)(run * RL) * N + w, tap, T, acc);
#pragma unroll
            for (int u = 0; u < RL; u++) {
                const long long uu = v0 + run * RL + u;
                if (uu < k2) out[uu * N + w] = acc[u];
            }
            if (t == ntiles - 1) {                            // the T newest spun vectors of the call -> history of the next one
                for (int e = tid; e < T * N; e += 256) {
                    const int tt = e / N, ch = e % N;
                    const long long vv = k2 - T + tt;         // >= v0 - (TPAD-1): the last tile holds vector k2-1 and T <= TPAD
                    hist[(size_t)ch * T + tt] = Sb[(size_t)(vv - v0 + TPAD - 1) * N + ch];
                }
            }
        }
        __syncthreads();
        // ---- D: keep the newest TPAD-1 rows for the next tile (through registers: source and destination overlap
        // when a tile is shorter than the history, e.g. 256 channels x 32 taps)
        {
            constexpr int ITER = ((TPAD - 1) * N + 255) / 256;
            float2 keep[ITER];
#pragma unroll
            for (int i = 0; i < ITER; i++) {
                const int e = tid + i * 256;
                keep[i] = e < (TPAD - 1) * N ? Sb[(size_t)OB * N + e] : make_float2(0.f, 0.f);
            }
            __syncthreads();
#pragma unroll
            for (int i = 0; i < ITER; i++) {
                const int e = tid + i * 256;
                if (e < (TPAD - 1) * N) Sb[e] = keep[i];
            }
        }
        __syncthreads();
    }
}

template <int LOG2N, int TPAD> constexpr size_t synth_fused_smem() {
    constexpr fftk::FftGeom G = fftk::fft_geom(LOG2N, 256);
    return ((size_t)G.n * (G.fpb + 1) + (size_t)G.fpb * G.np + (size_t)(TPAD - 1 + G.fpb) * G.n) * sizeof(float2);
}

template <int LOG2N, int TPAD, bool PADDED>
int32_t synth_fused_launch(b2s_synth *s, const float2 *in, long long in_stride, float2 *out, long long k2) {
    constexpr int OB = fftk::fft_geom(LOG2N, 256).fpb;
    constexpr size_t smem = synth_fused_smem<LOG2N, TPAD>();
    constexpr auto kern = synth_fused_kernel<LOG2N, TPAD, PADDED>;
    int resident = 1;
    B2S_TRY(smem_optin<kern>(s->ctx, smem, 256, &resident));
    constexpr int WARM = (TPAD - 1 + OB - 1) / OB;
    const long long ntiles = (k2 - (long long)WARM * OB + OB - 1) / OB;   // tiles over vectors [WARM*OB, k2)
    if (ntiles > 0x7fffff00ll) return b2s_fail(s->ctx, B2S_EUNSUPPORTED, "synthesizer: too many vectors in one call");
    const long long grid = std::min<long long>(ntiles, (long long)s->ctx->sm_count * resident);
    const long long tpc = (ntiles + grid - 1) / grid;
    const long long grid2 = (ntiles + tpc - 1) / tpc;         // no empty CTAs (the last tile must be owned by the last CTA)
    kern<<<(unsigned)grid2, 256, smem, s->ctx->stream>>>(in, in_stride, s->taps.arms_pad.get(), b2s_fft_twiddles(s->ifft.get()), out,
                                                          s->win.hist.get(), (int)s->T, k2, (int)ntiles, (int)tpc);
    B2S_CHECK_LAUNCH(s->ctx);
    return B2S_OK;
}

int synth_fused_ob(int log2n) { return fftk::fft_geom(log2n, 256).fpb; }
// vectors at the start of a call that stay on the generic path: the warm-up tiles of the first CTA
size_t synth_fused_lead(int log2n, int tpad) { const int ob = synth_fused_ob(log2n); return (size_t)((tpad - 1 + ob - 1) / ob) * ob; }

}  // namespace

extern "C" {

int32_t b2s_synth_plan_c32(b2s_ctx *ctx, size_t num_channels, const float *taps, size_t ntaps, b2s_synth **out) {
    if (!ctx || !out || !taps) return b2s_fail(ctx, B2S_EINVAL, "b2s_synth_plan_c32: NULL argument");
    *out = nullptr;
    if (num_channels < 2 || ntaps == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_synth_plan_c32: need >= 2 channels and taps");
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_synth> s(new b2s_synth());
    s->ctx = ctx; s->N = num_channels;
    const size_t N = s->N;
    std::vector<float> arms;
    const size_t T = pfb_partition(taps, ntaps, N, arms);
    s->T = T;
    b2s_fft *ifft = nullptr;
    B2S_TRY(b2s_fft_plan_c32(ctx, N, 1, 0, 0, 1.0f, &ifft));                  // plan_fft(n, Inverse) (synthesizer.rs:65)
    s->ifft.reset(ifft);
    const int tpad = getenv("B2S_SYNTH_NO_FUSED") ? 0 : pfb_fused_tpad(b2s_fft_log2n(ifft), T);
    B2S_TRY(s->taps.upload(ctx, arms, N, T, tpad, "synthesizer arms"));
    B2S_TRY(s->win.init(ctx, (int)N, (int)T, false, "synthesizer windows"));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *out = s.release();
    return B2S_OK;
}

void b2s_synth_destroy(b2s_synth *s) { PlanDeleter<b2s_synth>()(s); }

// One Kernel::work call (synthesizer.rs:80-144).  d_in is channel-major (stream w at d_in + w*in_stride),
// n_in the shortest input slice, d_out the single output slice of n_out_cap items.
int32_t b2s_synth_exec(b2s_synth *s, const void *d_in, size_t in_stride, size_t n_in, void *d_out, size_t n_out_cap,
                       size_t *consumed_per_channel, size_t *produced) {
    if (!s || !consumed_per_channel || !produced) return b2s_fail(s ? s->ctx : nullptr, B2S_EINVAL, "b2s_synth_exec: NULL argument");
    b2s_ctx *ctx = s->ctx;
    *consumed_per_channel = 0; *produced = 0;
    const size_t N = s->N, T = s->T;
    // closed form of `while n_in - c > 0 && (cap - p > N || !all_filled)`
    size_t k1 = 0, k2 = 0, p = 0;
    bool completes = false;
    const bool all_filled = s->win.full();
    if (!all_filled) {
        const size_t missing = s->win.missing() / N;          // vectors
        k1 = std::min(n_in, missing);
        completes = (k1 == missing) && k1 > 0;
        if (completes) p = N;                       // the completing vector writes its N outputs unconditionally
    }
    if (all_filled || completes) {
        const size_t remaining = n_in - k1;
        if (n_out_cap > p + N) {
            const size_t room = n_out_cap - N - p;  // vectors while cap - p > N  <=>  p < cap - N
            k2 = std::min(remaining, ceil_div(room, N));
        }
        p += k2 * N;
    }
    if (completes && n_out_cap < N)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_synth_exec: output slice (%zu) shorter than num_channels while the windows fill (the reference would index out of bounds)", n_out_cap);
    const size_t nv = k1 + k2;
    if (nv == 0) return B2S_OK;
    if (!d_in || (!d_out && p)) return b2s_fail(ctx, B2S_EINVAL, "b2s_synth_exec: NULL buffer");
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_synth_exec");
    // steady calls long enough for two tiles: the first OB vectors (their windows reach into the previous call's
    // history) through the three kernels below, everything after them through the fused kernel
    const int l2n = b2s_fft_log2n(s->ifft.get());
    const int tpad = s->taps.tpad;
    const size_t ob = tpad ? (size_t)synth_fused_ob(l2n) : 0;
    const size_t lead = tpad ? synth_fused_lead(l2n, tpad) : 0;
    const bool fused = tpad && all_filled && k1 == 0 && k2 >= lead + ob && k2 >= lead + T;
    const size_t k2_all = k2;
    if (fused) k2 = lead;                                 // the generic part
    const size_t items = (k1 + k2) * N;
    if (s->d_tmp.size() < 2 * items) B2S_TRY(s->d_tmp.reserve(ctx, 2 * (items * 5 / 4 + 1024), "synthesizer workspace"));
    float2 *vec = s->d_tmp.get(), *spun = s->d_tmp.get() + s->d_tmp.size() / 2;
    const size_t nvg = k1 + k2;                           // vectors of the generic part
    B2S_TRY(pfb_transpose(ctx, (const float2 *)d_in, vec, N, nvg, in_stride, N));   // vec[v * N + w] = in[w * in_stride + v]
    size_t fc = 0, fp = 0;
    int32_t rc = b2s_fft_exec(s->ifft.get(), vec, items, spun, items, &fc, &fp);
    if (rc != B2S_OK) return rc;
    B2S_TRY(s->win.push(ctx, spun, k1 * N));
    if (p) {
        const int u0 = completes ? -1 : 0;
        const size_t total = (k2 - (long long)u0) * N;
        const unsigned grid = (unsigned)std::min<size_t>(ceil_div(total, (size_t)256), (size_t)ctx->sm_count * 32);
        synth_bank_kernel<<<grid, 256, 0, ctx->stream>>>(spun + k1 * N, s->win.hist.get(), s->taps.arms.get(), (float2 *)d_out, (int)N, (int)T,
                                                         u0, (long long)k2);
        B2S_CHECK_LAUNCH(ctx);
    }
    if (fused) {
        // (the generic bank kernel above has read the old history; the fused kernel writes the new one)
        const int32_t frc = pfb_fused_dispatch(l2n, tpad, T, [&](auto L, auto P, auto D) {
            return synth_fused_launch<L, P, D>(s, (const float2 *)d_in, (long long)in_stride, (float2 *)d_out, (long long)k2_all);
        });
        if (frc != B2S_OK) return frc == B2S_EAGAIN ? b2s_fail(ctx, B2S_ESTATE, "synthesizer: fused shape mismatch") : frc;
    } else if (k2) {
        B2S_TRY(s->win.slide(ctx, spun + k1 * N, 0, (long long)(k2 * N)));
    }
    *consumed_per_channel = nv; *produced = p;
    return B2S_OK;
}

}  // extern "C"
