// pfb_common.cuh -- what the three polyphase filter-bank blocks (pfbarb.cu, chan.cu, synth.cu) share: the tap
// partition of pfb/utilities.rs:9-19, the reference's WindowBuffer (pfb/window_buffer.rs) over W windows, a strided
// transpose, and the scaffolding of the two fused steady-state kernels (chan_fused_kernel, synth_fused_kernel).
#pragma once
#include <algorithm>
#include <cmath>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "fft_common.cuh"

const float2 *b2s_fft_twiddles(const b2s_fft *p);   // fft.cu
int b2s_fft_log2n(const b2s_fft *p);

// partition_filter_taps: T = ceil(len as f32 / n as f32) taps per arm, arm i = taps[i::n] zero padded to T.
// Returns T and the arm-major table arms[i*T + j] = taps[i + j*n].
inline size_t pfb_partition(const float *taps, size_t ntaps, size_t n, std::vector<float> &arms) {
    const size_t T = (size_t)std::ceil((float)ntaps / (float)n);
    arms.assign(n * T, 0.0f);
    for (size_t i = 0; i < n; i++)
        for (size_t j = 0, idx = i; idx < ntaps; idx += n, j++) arms[i * T + j] = taps[idx];
    return T;
}

// ---- the reference's WindowBuffer, W windows of T samples -------------------------------------------------------
// Every window is created with pad_start = false and receives its pushes from one stream: item c of the stream goes to
// window c mod W (W-1 - c mod W when `mirror`: the channelizer walks its windows downwards) as that window's push
// number k = c / W.  A window's whole state is then k: push k finds start_idx = k mod T and num_samples_missing =
// max(T - k, 0), so while the window fills it writes slot (start_idx - missing) mod T = 2k mod T (window_buffer.rs:24-32:
// the first T samples land scattered, later ones overwrite earlier ones).  Once full, start_idx = T mod T = 0 and
// get_as_slice is slots [0, T): the fill writes straight into `hist`, which is then the window oldest sample first.
// Windows fill together: the stream fills all of them after exactly W*T items.
struct PfbWindows {
    Buf<float2> hist;              // [W][T], each window oldest sample first
    int W = 0, T = 0;
    bool mirror = false;
    size_t pushed = 0;             // items of the stream pushed so far while filling (W*T once full)

    int32_t init(b2s_ctx *ctx, int w, int t, bool mir, const char *what) {
        W = w; T = t; mirror = mir;
        if ((size_t)T * sizeof(float2) > ctx->smem_optin)      // slide() stages one window in shared memory
            return b2s_fail(ctx, B2S_EUNSUPPORTED, "%s: %d taps per window exceed the %zu bytes of shared memory a CTA can have",
                            what, T, ctx->smem_optin);
        B2S_TRY(hist.alloc(ctx, (size_t)W * T, what));
        return reset(ctx);
    }
    int32_t reset(b2s_ctx *ctx) {  // the reference's buffers start at zero; slots the fill skips stay zero
        pushed = 0;
        B2S_CUDA(ctx, cudaMemsetAsync(hist.get(), 0, hist.size() * sizeof(float2), ctx->stream));
        return B2S_OK;
    }
    bool full() const { return pushed == (size_t)W * T; }
    size_t missing() const { return (size_t)W * T - pushed; }
    // the fill: items pushed .. pushed+n of the stream are in[0, n), n <= missing()
    int32_t push(b2s_ctx *ctx, const float2 *in, size_t n);
    // steady state: item c0 + i of the stream is in[i] (only c0 mod W matters); window w becomes the last T items of
    // itself followed by the items that go to it
    int32_t slide(b2s_ctx *ctx, const float2 *in, long long c0, long long n);
};

namespace {

__device__ __forceinline__ int pfb_window_first(int W, int w, bool mirror, long long c0) {   // first r >= 0: c0 + r -> w
    const int q = mirror ? W - 1 - w : w;
    return (int)(((q - c0) % W + W) % W);
}

__global__ void pfb_push_kernel(float2 *hist, const float2 *__restrict__ in, int W, int T, bool mirror, long long c0,
                                long long n) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    float2 *h = hist + (size_t)w * T;
    for (long long r = pfb_window_first(W, w, mirror, c0); r < n; r += W) h[(2 * ((c0 + r) / W)) % T] = in[r];
}

__global__ void pfb_slide_kernel(float2 *hist, const float2 *__restrict__ in, int W, int T, bool mirror, long long c0,
                                 long long n) {
    extern __shared__ float2 tmp[];
    const int w = blockIdx.x;
    const long long r = pfb_window_first(W, w, mirror, c0);
    const long long m = n > r ? (n - 1 - r) / W + 1 : 0;     // items window w receives, the newest at in[c_new]
    const long long c_new = r + (m - 1) * W;
    float2 *h = hist + (size_t)w * T;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const long long j = T - 1 - t;                       // new h[t] = the j-th newest
        tmp[t] = j < m ? in[c_new - j * W] : h[t + m];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) h[t] = tmp[t];
}

// dst[c * ldd + r] = src[r * lds + c] for r < rows, c < cols: 32 x 32 tiles through shared memory, coalesced on both
// sides.  One CTA of 32 x 8 threads per tile, row tiles first.
__global__ void pfb_transpose_kernel(const float2 *__restrict__ src, float2 *__restrict__ dst, long long rows,
                                     long long cols, long long lds, long long ldd) {
    __shared__ float2 tile[32][33];
    const long long rt = (rows + 31) / 32;
    const long long r0 = (long long)(blockIdx.x % rt) * 32, c0 = (long long)(blockIdx.x / rt) * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const long long r = r0 + i, c = c0 + threadIdx.x;
        if (r < rows && c < cols) tile[i][threadIdx.x] = src[r * lds + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const long long r = r0 + threadIdx.x, c = c0 + i;
        if (r < rows && c < cols) dst[c * ldd + r] = tile[threadIdx.x][i];
    }
}

}  // namespace

inline int32_t PfbWindows::push(b2s_ctx *ctx, const float2 *in, size_t n) {
    if (!n) return B2S_OK;
    pfb_push_kernel<<<(unsigned)ceil_div((size_t)W, 128), 128, 0, ctx->stream>>>(hist.get(), in, W, T, mirror,
                                                                                (long long)pushed, (long long)n);
    B2S_CHECK_LAUNCH(ctx);
    pushed += n;
    return B2S_OK;
}

inline int32_t PfbWindows::slide(b2s_ctx *ctx, const float2 *in, long long c0, long long n) {
    const size_t bytes = (size_t)T * sizeof(float2);   // one window in shared memory: above 48 KiB (T > 6144) only opted in
    if (bytes > 48 * 1024) B2S_TRY(smem_optin<pfb_slide_kernel>(ctx, ctx->smem_optin));
    pfb_slide_kernel<<<(unsigned)W, 64, bytes, ctx->stream>>>(hist.get(), in, W, T, mirror, c0, n);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

inline int32_t pfb_transpose(b2s_ctx *ctx, const float2 *src, float2 *dst, size_t rows, size_t cols, size_t lds, size_t ldd) {
    const unsigned grid = (unsigned)(ceil_div(rows, 32) * ceil_div(cols, 32));
    pfb_transpose_kernel<<<grid, dim3(32, 8), 0, ctx->stream>>>(src, dst, (long long)rows, (long long)cols, (long long)lds,
                                                                (long long)ldd);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

// ---- fused steady-state kernels of the channelizer and the synthesizer ------------------------------------------
// Both serve N a power of two in [4, 256] and T <= 32, with T padded to TPAD = 8, 16 or 32 zero taps beyond T (older
// samples).  pfb_fused_tpad: that TPAD, 0 outside these shapes.
inline int pfb_fused_tpad(int log2n, size_t T) {
    if (log2n < 2 || log2n > 8 || T > 32) return 0;
    return T <= 8 ? 8 : (T <= 16 ? 16 : 32);
}

// f(L, P, D) with L = log2n, P = tpad and D = (T < tpad) as std::integral_constant: the instantiations of a fused kernel;
// B2S_EAGAIN for a shape outside them
template <typename F> int32_t pfb_fused_dispatch(int log2n, int tpad, size_t T, F &&f) {
    auto at = [&](auto P) {
        return fftk::with_log2n<2, 8>(log2n, B2S_EAGAIN, [&](auto L) {
            return T < (size_t)tpad ? f(L, P, std::true_type{}) : f(L, P, std::false_type{});
        });
    };
    switch (tpad) {
        case 8: return at(std::integral_constant<int, 8>{});
        case 16: return at(std::integral_constant<int, 16>{});
        case 32: return at(std::integral_constant<int, 32>{});
        default: return B2S_EAGAIN;
    }
}

// The tap tables of a channelizer or synthesizer bank, tap-major so that adjacent windows -- which meet adjacent arms --
// read adjacent floats: arms [T][N], arms[j*N + i] = arm_i[j] (newest sample <-> j = 0), and for the fused kernel the
// same zero-padded to [tpad][N].
struct PfbBankTaps {
    Buf<float> arms, arms_pad;
    int tpad = 0;

    // arm_major: pfb_partition's [N][T]; waits for the uploads
    int32_t upload(b2s_ctx *ctx, const std::vector<float> &arm_major, size_t N, size_t T, int fused_tpad, const char *what) {
        tpad = fused_tpad;
        std::vector<float> tm(std::max<size_t>(T, (size_t)tpad) * N, 0.0f);
        for (size_t i = 0; i < N; i++)
            for (size_t j = 0; j < T; j++) tm[j * N + i] = arm_major[i * T + j];
        B2S_TRY(arms.upload(ctx, tm.data(), T * N, what));
        if (tpad) B2S_TRY(arms_pad.upload(ctx, tm.data(), (size_t)tpad * N, what));
        B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return B2S_OK;
    }
};

// One thread's column of a fused bank: col[k * N], k < RL + TPAD - 1, are consecutive samples of its window, oldest
// first; output u of the run is the window ending at row u + TPAD - 1 with tap j on its j-th newest sample.  The column
// is streamed through registers once and every sample is multiplied into each output that contains it (taps in
// registers, static indices after unrolling), so every output accumulates oldest sample first like the reference.
// PADDED (T < TPAD): the padded taps j >= T are skipped, not multiplied -- 0 * inf is NaN, and a non-finite sample must
// reach exactly the T outputs it reaches in the reference.  Unpadded banks (T == TPAD) are compiled without the guard.
template <int N, int RL, int TPAD, bool PADDED>
__device__ __forceinline__ void pfb_bank_column(const float2 *col, const float (&tap)[TPAD], int T, float2 (&acc)[RL]) {
#pragma unroll
    for (int u = 0; u < RL; u++) acc[u] = make_float2(0.f, 0.f);
#pragma unroll
    for (int k = 0; k < RL + TPAD - 1; k++) {
        const float2 x = col[(size_t)k * N];
#pragma unroll
        for (int u = 0; u < RL; u++) {
            const int j = u + TPAD - 1 - k;          // output u sees this row as its j-th newest sample
            if (j >= 0 && j < TPAD && (!PADDED || j < T)) mac(acc[u], x, tap[j]);
        }
    }
}
