// fft.cu -- batched power-of-two Complex<f32> FFT, one pass through shared memory (sm_90a).
//
// Device version of the reference's Fft block (src/blocks/fft.rs:160-221), whose arithmetic is
// rustfft 6.4 (crates.io): forward X[k] = sum_n x[n] e^{-2 pi i kn/N}, inverse un-normalised
// e^{+...}; optional fftshift (after a forward transform fft.rs:196-204, before an inverse one
// :179-185) and optional scalar normalisation (:206-210).
//
// Algorithm: Stockham autosort, mixed radix 16/8/4/2 butterflies held in registers; a transform
// lives in shared memory between passes (padded: idx + idx/16, so the stride-R scatter of the
// first pass is bank-conflict free), the first pass reads global memory and the last pass
// writes it, both fully coalesced (element j + r*N/R for consecutive j).  HBM traffic is the
// algorithmic minimum, 8 B in + 8 B out per sample (the reference's WGSL/CubeCL prior art makes
// one global pass per radix-2 stage, perf/burn/src/bin/fft-wgpu-hack.rs:270-397).
// The passes are fftk::fft_passes (fft_common.cuh); this file supplies their first load and last
// store.  fftshift is an index rotation on the first-pass load / last-pass store, normalisation a
// multiply on the store; the inverse transform is conj(FFT(conj(x))) (conjugations are free on
// load/store).  Twiddles come from a table W_N[k] evaluated in f64 on the host.
#include <cmath>
#include <cstdlib>

#include "common.cuh"
#include "fft_common.cuh"

namespace {

using namespace fftk;

struct FftArgs {
    const float2 *in;
    float2 *out;
    const float2 *tw;
    long long nfft;
    int inverse, shift, has_norm;
    float norm;
};

constexpr int kFftThreads = 256;

// CTA size and CTAs per SM the register allocation must allow, per size.  <= 4096: three 256-thread CTAs per SM --
// naming a minimum of 1 lets ptxas take more registers than three CTAs allow.  8192: the unconstrained build takes one
// 256-thread CTA per SM by registers although shared memory admits more -> cap at 128 registers, two CTAs.  16384: one
// transform = one CTA = one SM (139 KiB of shared memory); 1024 threads run ONE butterfly each per pass at 64 registers
// and give the SM 32 warps to hide latency with.
constexpr int fft_cta_threads(int log2n) { return log2n == 14 ? 1024 : kFftThreads; }
constexpr int fft_min_blocks(int log2n) { return log2n == 14 ? 1 : (log2n == 13 ? 2 : 3); }

template <int LOG2N, int TH, int MINB>
__global__ void __launch_bounds__(TH, MINB) fft_kernel(const FftArgs a) {
    constexpr FftGeom G = fft_geom(LOG2N, TH);
    constexpr int N = G.n;
    extern __shared__ __align__(16) unsigned char fsm[];
    const int t = threadIdx.x % G.t, fl = threadIdx.x / G.t;
    const long long f = (long long)blockIdx.x * G.fpb + fl;
    const bool active = f < a.nfft;
    float2 *sm = reinterpret_cast<float2 *>(fsm) + (size_t)fl * G.np;
    // idle transform slots of the last CTA recompute transform nfft-1 and skip the store
    const long long fc = active ? f : a.nfft - 1;
    const float2 *gin = a.in + fc * N;
    float2 *gout = a.out + fc * N;
    // twiddles from the table after each barrier: fetching them a pass ahead costs registers and spills at 8192/16384.
    // The last pass stores to global memory and ends the kernel: it runs without barriers.
    fft_passes<LOG2N, G.t, Tw::Table>(
        [&](int idx) {
            // inverse + shift: buff[k] = i[(k + N/2) % N]   (fft.rs:179-185)
            const int src = (a.inverse && a.shift) ? ((idx + N / 2) & (N - 1)) : idx;
            float2 x = __ldg(gin + src);
            if (a.inverse) x.y = -x.y;
            return x;
        },
        [&](int idx, float2 y) {
            if (a.inverse) y.y = -y.y;
            if (a.has_norm) { y.x *= a.norm; y.y *= a.norm; }
            // forward + shift: o[k] = X[(k + N/2) % N]   (fft.rs:196-204)
            const int dst = (!a.inverse && a.shift) ? ((idx + N / 2) & (N - 1)) : idx;
            if (active) gout[dst] = y;
        },
        sm, a.tw, t, false, false);
}

template <int LOG2N>
int32_t launch_fft(b2s_fft *p, const FftArgs &a, cudaStream_t stream) {
    constexpr int TH = fft_cta_threads(LOG2N);
    constexpr FftGeom G = fft_geom(LOG2N, TH);
    constexpr size_t smem = (size_t)G.fpb * G.np * sizeof(float2);
    constexpr auto kern = fft_kernel<LOG2N, TH, fft_min_blocks(LOG2N)>;
    B2S_TRY(smem_optin<kern>(p->ctx, smem));
    const unsigned grid = (unsigned)ceil_div((size_t)a.nfft, (size_t)G.fpb);
    kern<<<grid, TH, smem, stream>>>(a);
    B2S_CHECK_LAUNCH(p->ctx);
    return B2S_OK;
}


// ---- Bluestein: X[k] = w[k] * sum_n (x[n] w[n]) * conj(w[k-n]),  w[n] = exp(-i pi n^2 / N) ----------
// One transform per thread group: a = x.w zero-padded to M, A = FFT_M(a), C = A . Bhat,
// c = IFFT_M(C), X = c . w -- all inside one kernel with the M-point buffer in shared memory.
struct BsArgs {
    const float2 *in;
    float2 *out;
    const float2 *tw, *chirp, *bhat;
    long long nfft;
    int n, inverse, shift, has_norm;
    float norm;
};

template <int LOG2M>
__global__ void __launch_bounds__(kFftThreads) bluestein_kernel(const BsArgs a) {
    constexpr FftGeom G = fft_geom(LOG2M, kFftThreads);
    extern __shared__ __align__(16) unsigned char fsm[];
    const int t = threadIdx.x % G.t, fl = threadIdx.x / G.t;
    const long long f = (long long)blockIdx.x * G.fpb + fl;
    const bool active = f < a.nfft;
    const long long fc = active ? f : a.nfft - 1;
    float2 *sm = reinterpret_cast<float2 *>(fsm) + (size_t)fl * G.np;
    const float2 *gin = a.in + fc * a.n;
    float2 *gout = a.out + fc * a.n;
    const int n = a.n, half = n / 2;
    auto st_sm = [&](int idx, float2 v) { sm[pad(idx)] = v; };
    // forward M-point FFT of a[j] = x'[j] * w[j]  (x' = conj / pre-shifted input for the inverse direction)
    fft_passes<LOG2M, G.t, Tw::Ahead>(
        [&](int idx) {
            if (idx >= n) return make_float2(0.f, 0.f);
            const int src = (a.inverse && a.shift) ? (idx + half) % n : idx;        // fft.rs:179-185
            float2 x = __ldg(gin + src);
            if (a.inverse) x.y = -x.y;
            return cmul(x, __ldg(a.chirp + idx));
        },
        st_sm, sm, a.tw, t, false);
    // inverse M-point FFT of A . Bhat as conj(FFT(conj(.))), then the post-chirp
    fft_passes<LOG2M, G.t, Tw::Ahead>(
        [&](int idx) {
            const float2 y = cmul(sm[pad(idx)], __ldg(a.bhat + idx));
            return make_float2(y.x, -y.y);
        },
        [&](int idx, float2 v) {
            if (idx >= n || !active) return;
            float2 y = cmul(make_float2(v.x, -v.y), __ldg(a.chirp + idx));
            if (a.inverse) y.y = -y.y;
            if (a.has_norm) { y.x *= a.norm; y.y *= a.norm; }
            const int dst = (!a.inverse && a.shift) ? (idx + n - half) % n : idx;   // o[k] = X[(k + n/2) % n]  (fft.rs:196-204)
            gout[dst] = y;
        },
        sm, a.tw, t, true);
}

template <int LOG2M>
int32_t launch_bluestein(b2s_fft *p, const BsArgs &a, cudaStream_t stream) {
    constexpr FftGeom G = fft_geom(LOG2M, kFftThreads);
    constexpr size_t smem = (size_t)G.fpb * G.np * sizeof(float2);
    constexpr auto kern = bluestein_kernel<LOG2M>;
    B2S_TRY(smem_optin<kern>(p->ctx, smem));
    const unsigned grid = (unsigned)ceil_div((size_t)a.nfft, (size_t)G.fpb);
    kern<<<grid, kFftThreads, smem, stream>>>(a);
    B2S_CHECK_LAUNCH(p->ctx);
    return B2S_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// LARGE transforms: rustfft plans any length (src/blocks/fft.rs:98-103); beyond what one shared-memory transform holds
// the classic four-step algorithm runs through HBM:  M = n1 * n2,  i = i1*n2 + i2,  k = k1 + n1*k2,
//   X[k1 + n1*k2] = sum_{i2} W_{n2}^{i2 k2} * ( W_M^{i2 k1} * sum_{i1} x[i1*n2 + i2] W_{n1}^{i1 k1} )
// as  transpose -> n2 transforms of length n1 -> twiddle + transpose -> n1 transforms of length n2 -> transpose,
// every transform being the batched shared-memory kernel above.  Five passes over the data instead of one: this path
// exists for completeness (spectrum analysers with 64 Ki+ bins, odd lengths), not for speed.
// ---------------------------------------------------------------------------------------------------------------
struct BigT {                 // dst[c * R + r] = f(src[r * C + c]) with optional index rotations / twiddle / scale
    const float2 *src;
    float2 *dst;
    long long R, C, M;
    int conj_in, conj_out, twiddle;
    long long src_rot, dst_rot;   // src index (idx + src_rot) % M ; dst index (idx + dst_rot) % M
    float scale;
};

__global__ void big_transpose_kernel(const BigT a) {
    __shared__ float2 tile[32][33];
    const long long r0 = (long long)blockIdx.y * 32, c0 = (long long)blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const long long r = r0 + i, c = c0 + threadIdx.x;
        if (r < a.R && c < a.C) {
            long long idx = r * a.C + c;
            if (a.src_rot) { idx += a.src_rot; if (idx >= a.M) idx -= a.M; }
            float2 v = a.src[idx];
            if (a.conj_in) v.y = -v.y;
            if (a.twiddle) {                                  // W_M^{r c}, exponent reduced exactly, angle in f64
                const unsigned long long t = ((unsigned long long)r * (unsigned long long)c) % (unsigned long long)a.M;
                double sn, cs;
                sincospi(-2.0 * (double)t / (double)a.M, &sn, &cs);
                const float wr = (float)cs, wi = (float)sn;
                v = make_float2(v.x * wr - v.y * wi, v.x * wi + v.y * wr);
            }
            tile[i][threadIdx.x] = v;
        }
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const long long c = c0 + i, r = r0 + threadIdx.x;
        if (r < a.R && c < a.C) {
            float2 v = tile[threadIdx.x][i];
            if (a.conj_out) v.y = -v.y;
            v.x *= a.scale; v.y *= a.scale;
            long long idx = c * a.R + r;
            if (a.dst_rot) { idx += a.dst_rot; if (idx >= a.M) idx -= a.M; }
            a.dst[idx] = v;
        }
    }
}

int32_t big_transpose(b2s_ctx *ctx, const BigT &a, cudaStream_t st) {
    dim3 grid((unsigned)ceil_div((size_t)a.C, (size_t)32), (unsigned)ceil_div((size_t)a.R, (size_t)32));
    big_transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(a);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

// Bluestein element-wise stages for M > 16384
__global__ void big_bs_pre(const float2 *__restrict__ in, const float2 *__restrict__ chirp, float2 *a, long long n, long long M,
                           int inverse, long long src_rot) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < M; j += stride) {
        float2 v = make_float2(0.f, 0.f);
        if (j < n) {
            long long sidx = j + src_rot; if (sidx >= n) sidx -= n;
            float2 x = in[sidx];
            if (inverse) x.y = -x.y;
            v = cmul(x, chirp[j]);
        }
        a[j] = v;
    }
}
__global__ void big_bs_mul(float2 *A, const float2 *__restrict__ bhat, long long M) {   // A <- conj(A . Bhat): input of the inverse M-point FFT
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < M; j += stride) {
        const float2 y = cmul(A[j], bhat[j]);
        A[j] = make_float2(y.x, -y.y);
    }
}
__global__ void big_bs_post(const float2 *__restrict__ c, const float2 *__restrict__ chirp, float2 *out, long long n, int inverse,
                            long long dst_rot, float scale) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride) {
        float2 y = cmul(make_float2(c[k].x, -c[k].y), chirp[k]);      // conj closes the inverse M-point FFT
        if (inverse) y.y = -y.y;
        y.x *= scale; y.y *= scale;
        long long d = k + dst_rot; if (d >= n) d -= n;
        out[d] = y;
    }
}

// plan internals for the kernels that embed an N-point transform (chan.cu's fused channelizer)
const float2 *b2s_fft_twiddles(const b2s_fft *p) { return p ? p->d_tw.get() : nullptr; }
int b2s_fft_log2n(const b2s_fft *p) { return (p && !p->bluestein && !p->big) ? p->log2n : -1; }

// one M-point forward transform src -> dst through the four-step scratch (d_work[0 .. 2M))
static int32_t big_fft(b2s_fft *p, const float2 *src, float2 *dst, int conj_in, int conj_out, long long src_rot,
                       long long dst_rot, float scale, cudaStream_t st) {
    b2s_ctx *ctx = p->ctx;
    const long long M = (long long)p->big_m, n1 = (long long)p->big_n1, n2 = (long long)p->big_n2;
    float2 *A = p->d_work.get(), *B = p->d_work.get() + M;
    size_t c = 0, q = 0;
    int32_t rc;
    BigT t{};
    t.M = M; t.scale = 1.0f;
    t.src = src; t.dst = A; t.R = n1; t.C = n2; t.conj_in = conj_in; t.src_rot = src_rot;       // x[i1][i2] -> A[i2][i1]
    if ((rc = big_transpose(ctx, t, st))) return rc;
    if ((rc = b2s_fft_exec(p->sub1.get(), A, (size_t)M, B, (size_t)M, &c, &q))) return rc;               // n2 transforms of length n1
    t = BigT{}; t.M = M; t.scale = 1.0f;
    t.src = B; t.dst = A; t.R = n2; t.C = n1; t.twiddle = 1;                                       // Y[i2][k1] W_M^{i2 k1} -> A[k1][i2]
    if ((rc = big_transpose(ctx, t, st))) return rc;
    if ((rc = b2s_fft_exec(p->sub2.get(), A, (size_t)M, B, (size_t)M, &c, &q))) return rc;               // n1 transforms of length n2
    t = BigT{}; t.M = M;
    t.src = B; t.dst = dst; t.R = n1; t.C = n2; t.conj_out = conj_out; t.dst_rot = dst_rot; t.scale = scale;   // Z[k1][k2] -> X[k2*n1 + k1]
    return big_transpose(ctx, t, st);
}

extern "C" {

int32_t b2s_fft_plan_c32(b2s_ctx *ctx, size_t n, int32_t inverse, int32_t fft_shift, int32_t has_normalize,
                         float normalize, b2s_fft **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_fft_plan_c32: NULL argument");
    *out = nullptr;
    if (n < 2) return b2s_fail(ctx, B2S_EINVAL, "b2s_fft_plan_c32: n must be >= 2");
    const bool pow2 = (n & (n - 1)) == 0;
    // one transform in shared memory up to 16384 points (Bluestein: M >= 2n-1 <= 16384); beyond that four-step
    // through HBM, bounded by the scratch it needs (2 M / 4 M items)
    const bool big = pow2 ? n > 16384 : n > 8192;
    if (pow2 && n > ((size_t)1 << 26)) return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_fft_plan_c32: n = %zu > 2^26", n);
    if (!pow2 && n > ((size_t)1 << 24)) return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_fft_plan_c32: non-power-of-two n = %zu > 2^24", n);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_fft> p(new b2s_fft());
    p->ctx = ctx; p->n = n; p->big = big;
    p->inverse = inverse != 0; p->shift = fft_shift != 0; p->has_norm = has_normalize != 0; p->norm = normalize;
    const double PI = 3.14159265358979323846264338327950288;
    size_t tw_n = n;
    if (pow2) {
        while (((size_t)1 << p->log2n) < n) p->log2n++;
    } else {
        p->bluestein = true;
        while (((size_t)1 << p->log2m) < 2 * n - 1) p->log2m++;
        tw_n = (size_t)1 << p->log2m;
    }
    if (big) {
        // M = n1 * n2 with both factors <= 16384; the two shared-memory plans do the actual transforms
        p->big_m = tw_n;
        int l2 = 0;
        while (((size_t)1 << l2) < tw_n) l2++;
        p->big_n1 = (size_t)1 << ((l2 + 1) / 2);
        p->big_n2 = tw_n / p->big_n1;
        b2s_fft *sub = nullptr;
        B2S_TRY(b2s_fft_plan_c32(ctx, p->big_n1, 0, 0, 0, 1.0f, &sub));
        p->sub1.reset(sub);
        B2S_TRY(b2s_fft_plan_c32(ctx, p->big_n2, 0, 0, 0, 1.0f, &sub));
        p->sub2.reset(sub);
        B2S_TRY(p->d_work.alloc(ctx, (p->bluestein ? 4 : 2) * tw_n, "fft four-step scratch"));
    }
    const std::vector<float2> tw = twiddle_table(big ? 1 : tw_n);   // four-step: W_1 = {1}, unused
    B2S_TRY(p->d_tw.upload(ctx, tw.data(), tw.size(), "fft twiddles"));
    std::vector<float2> chirp, bhat;
    if (p->bluestein) {
        const size_t M = tw_n;
        chirp.resize(n); bhat.resize(M);
        std::vector<double> br(M, 0.0), bi(M, 0.0);
        for (size_t k = 0; k < n; k++) {
            const unsigned long long k2 = ((unsigned long long)k * k) % (2ull * n);     // k^2 mod 2n, exact
            const double ang = -PI * (double)k2 / (double)n;
            chirp[k] = make_float2((float)std::cos(ang), (float)std::sin(ang));
            br[k] = std::cos(ang); bi[k] = -std::sin(ang);                             // conj(w[k])
            if (k) { br[M - k] = br[k]; bi[M - k] = bi[k]; }
        }
        // Bhat = FFT_M(b) / M in f64 (iterative radix-2), once per plan
        std::vector<double> xr(br), xi(bi);
        for (size_t i = 1, j = 0; i < M; i++) {
            size_t bit = M >> 1;
            for (; j & bit; bit >>= 1) j ^= bit;
            j ^= bit;
            if (i < j) { std::swap(xr[i], xr[j]); std::swap(xi[i], xi[j]); }
        }
        for (size_t len = 2; len <= M; len <<= 1)
            for (size_t j = 0; j < len / 2; j++) {
                const double ang = -2.0 * PI * (double)j / (double)len, wr = std::cos(ang), wi = std::sin(ang);
                for (size_t s0 = 0; s0 < M; s0 += len) {
                    const size_t u = s0 + j, v = u + len / 2;
                    const double tr = xr[v] * wr - xi[v] * wi, ti = xr[v] * wi + xi[v] * wr;
                    xr[v] = xr[u] - tr; xi[v] = xi[u] - ti; xr[u] += tr; xi[u] += ti;
                }
            }
        for (size_t k = 0; k < M; k++) bhat[k] = make_float2((float)(xr[k] / (double)M), (float)(xi[k] / (double)M));
        B2S_TRY(p->d_chirp.upload(ctx, chirp.data(), n, "fft bluestein chirp"));
        B2S_TRY(p->d_bhat.upload(ctx, bhat.data(), M, "fft bluestein kernel"));
    }
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *out = p.release();
    return B2S_OK;
}

void b2s_fft_destroy(b2s_fft *p) { PlanDeleter<b2s_fft>()(p); }

size_t b2s_fft_length(const b2s_fft *p) { return p ? p->n : 0; }

int32_t b2s_fft_exec(b2s_fft *p, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                     size_t *consumed, size_t *produced) {
    if (!p || !consumed || !produced) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_fft_exec: NULL argument");
    // m = min(i.len(), o.len()) rounded down to a multiple of len (fft.rs:169-170)
    size_t m = n_in < n_out_cap ? n_in : n_out_cap;
    m = (m / p->n) * p->n;
    *consumed = m; *produced = m;
    if (m == 0) return B2S_OK;
    if (!d_in || !d_out) return b2s_fail(p->ctx, B2S_EINVAL, "b2s_fft_exec: NULL buffer");
    if (d_in == d_out) return b2s_fail(p->ctx, B2S_EINVAL, "b2s_fft_exec: in-place is not supported");
    DeviceGuard g(p->ctx->device);
    NvtxRange nvtx("b2s_fft_exec");
    if (p->big) {
        cudaStream_t st = p->ctx->stream;
        const long long n = (long long)p->n, M = (long long)p->big_m, half = n / 2;
        const float scale = p->has_norm ? p->norm : 1.0f;
        const int gridE = p->ctx->sm_count * 8;
        for (size_t fr = 0; fr < m / p->n; fr++) {
            const float2 *in = (const float2 *)d_in + fr * p->n;
            float2 *out = (float2 *)d_out + fr * p->n;
            int32_t rc;
            if (!p->bluestein) {
                // inverse = conj o FFT o conj; shift: pre-rotation for the inverse, post-rotation for the forward transform
                rc = big_fft(p, in, out, p->inverse, p->inverse, (p->inverse && p->shift) ? half : 0,
                             (!p->inverse && p->shift) ? half : 0, scale, st);
                if (rc) return rc;
                continue;
            }
            float2 *b0 = p->d_work.get() + 2 * M, *b1 = p->d_work.get() + 3 * M;
            big_bs_pre<<<gridE, 256, 0, st>>>(in, p->d_chirp.get(), b0, n, M, p->inverse, (p->inverse && p->shift) ? half : 0);
            B2S_CHECK_LAUNCH(p->ctx);
            if ((rc = big_fft(p, b0, b1, 0, 0, 0, 0, 1.0f, st))) return rc;
            big_bs_mul<<<gridE, 256, 0, st>>>(b1, p->d_bhat.get(), M);
            B2S_CHECK_LAUNCH(p->ctx);
            if ((rc = big_fft(p, b1, b0, 0, 0, 0, 0, 1.0f, st))) return rc;
            big_bs_post<<<gridE, 256, 0, st>>>(b0, p->d_chirp.get(), out, n, p->inverse, (!p->inverse && p->shift) ? n - half : 0, scale);
            B2S_CHECK_LAUNCH(p->ctx);
        }
        return B2S_OK;
    }
    if (p->bluestein) {
        BsArgs b;
        b.in = (const float2 *)d_in; b.out = (float2 *)d_out; b.tw = p->d_tw.get(); b.chirp = p->d_chirp.get(); b.bhat = p->d_bhat.get();
        b.nfft = (long long)(m / p->n); b.n = (int)p->n;
        b.inverse = p->inverse; b.shift = p->shift; b.has_norm = p->has_norm; b.norm = p->norm;
        const int rc = with_log2n<2, 14>(p->log2m, B2S_EUNSUPPORTED, [&](auto L) { return launch_bluestein<L>(p, b, p->ctx->stream); });
        return rc == B2S_EUNSUPPORTED ? b2s_fail(p->ctx, rc, "b2s_fft_exec: unsupported Bluestein size") : rc;
    }
    FftArgs a;
    a.in = (const float2 *)d_in; a.out = (float2 *)d_out; a.tw = p->d_tw.get(); a.nfft = (long long)(m / p->n);
    a.inverse = p->inverse; a.shift = p->shift; a.has_norm = p->has_norm; a.norm = p->norm;
    const int rc = with_log2n<1, 14>(p->log2n, B2S_EUNSUPPORTED, [&](auto L) { return launch_fft<L>(p, a, p->ctx->stream); });
    return rc == B2S_EUNSUPPORTED ? b2s_fail(p->ctx, rc, "b2s_fft_exec: unsupported size") : rc;
}

}  // extern "C"
