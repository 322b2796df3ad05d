// chan.cu -- polyphase channelizer (src/blocks/pfb/channelizer.rs:88-223) on the device:
// SURVEY.md §8f row 2, a pure composition of the FIR-bank and FFT pieces of the hot path.
//
// Reference semantics restated: every consumed sample is pushed into window `base_index`, which
// then decrements modulo N -- so window w holds the stream decimated by N at phase (base0 - w);
// after each group of D = N / oversample_rate pushes, arm i (taps[i::N]) filters window
// (base_index + i + 1) % N into fft_buf[that window], an un-normalised inverse FFT over the N
// buffers de-spins, and element ch goes to output stream ch.
//   * start-up: windows fill through WindowBuffer::push, which scatters the first T samples of a
//     window (window_buffer.rs:24-32), and the call in which the last window fills returns
//     WITHOUT consuming (channelizer.rs:170-180), so those samples are pushed a second time.
//     Both are reproduced: a one-thread kernel replays the pushes on the data, the host mirrors
//     the bookkeeping (it is data-independent).
//   * steady state is closed-form: one thread per (output vector o, window b) gathers the T newest
//     samples of its phase (history buffer + this call's input) and dots them with its arm; the
//     N-point inverse FFT is the batched FFT kernel of fft.cu (any N: radix or Bluestein), a
//     transposing store writes channel-major output streams.
#include <cmath>
#include <cstdlib>

#include "common.cuh"
#include "fft_common.cuh"

const float2 *b2s_fft_twiddles(const b2s_fft *p);   // fft.cu
int b2s_fft_log2n(const b2s_fft *p);

struct b2s_chan {
    b2s_ctx *ctx = nullptr;
    size_t N = 0, D = 0, T = 0;
    Buf<float> d_arms;              // [T][N] (tap-major): d_arms[j*N + i] = arm_i[j] = taps[i + j*N] (utilities.rs:9-19;
                                    // newest sample <-> j = 0).  Tap-major so that adjacent windows -- which meet
                                    // adjacent arms -- read adjacent floats (arm-major cost 32 L1 lines per warp load)
    Buf<float2> d_circ;             // [N][2T] circular windows (used while filling)
    Buf<float2> d_hist;             // [N][T] windows in time order once filled
    Buf<int> d_wstate;              // [2N]: start_idx[N], missing[N]
    std::vector<int> start_idx, missing;   // host mirror of the WindowBuffer bookkeeping
    size_t base_index = 0;
    bool all_filled = false;
    PlanPtr<b2s_fft> ifft;
    Buf<float2> d_tmp;              // two halves: bank outputs, spectra
    Buf<float> d_arms_pad;          // [TPAD][N]: d_arms zero-padded to the fused kernel's tap count
    int tpad = 0;
};

namespace {

__global__ void chan_fill_kernel(const float2 *__restrict__ in, float2 *circ, int *wstate, int N, int T,
                                 int base_index, int count) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    int *start = wstate, *missing = wstate + N;
    for (int c = 0; c < count; c++) {
        const int w = base_index;
        int idx = (start[w] - missing[w]) % T;
        if (idx < 0) idx += T;
        float2 *cw = circ + (size_t)w * 2 * T;
        cw[idx] = in[c]; cw[idx + T] = in[c];
        if (missing[w] > 0) missing[w]--;
        start[w] = (start[w] + 1) % T;
        base_index = base_index == 0 ? N - 1 : base_index - 1;
    }
}

__global__ void chan_hist_from_circ(const float2 *__restrict__ circ, const int *__restrict__ wstate, float2 *hist,
                                    int N, int T) {
    const int w = blockIdx.x;
    const int s = wstate[w];
    for (int t = threadIdx.x; t < T; t += blockDim.x) hist[(size_t)w * T + t] = circ[(size_t)w * 2 * T + s + t];
}

// Critically sampled steady state (D == N, the window already holds T samples of this call): every output
// pushes exactly one new sample into every window and the window keeps meeting the same arm, so the T samples
// and the T taps live in REGISTERS; the output loop is unrolled T times so that the ring positions are static.
// Per output: one 8-byte load, 2*T FMAs, one store (the general loop below re-reads all T samples and taps).
// MAC order is unchanged: oldest sample first.
template <int TT>
__device__ __forceinline__ void chan_run_regs(const float2 *__restrict__ in, const float *__restrict__ a /*arm, tap j at a[j*N]*/,
                                              float2 *__restrict__ fftbuf, int N, int b, long long c_new,
                                              long long o_begin, long long o_end) {
    float2 w[TT];                                   // slot k holds the sample of age (TT-1-k) at the start of a group
    float tr[TT];
#pragma unroll
    for (int k = 0; k < TT; k++) {
        w[k] = __ldg(in + (c_new - (long long)(TT - 1 - k) * N));
        tr[k] = __ldg(a + (size_t)k * N);
    }
    // q[u]: the sample output o+u pushes for output o+u+1 -- fetched one whole group (TT outputs) ahead so that a
    // DRAM/L2 round trip is paid once per TT outputs and overlaps TT*2*TT FMAs
    const float2 *nxt = in + c_new + N;
    float2 q[TT];
#pragma unroll
    for (int u = 0; u < TT; u++) q[u] = (o_begin + u + 1 < o_end) ? __ldg(nxt + (long long)u * N) : make_float2(0.f, 0.f);
    for (long long o = o_begin; o < o_end; o += TT) {
        float2 qn[TT];
#pragma unroll
        for (int u = 0; u < TT; u++)
            qn[u] = (o + TT + u + 1 < o_end) ? __ldg(nxt + (long long)(TT + u) * N) : make_float2(0.f, 0.f);
        nxt += (long long)TT * N;
#pragma unroll
        for (int u = 0; u < TT; u++) {
            if (o + u < o_end) {
                float re = 0.f, im = 0.f;
#pragma unroll
                for (int j = TT - 1; j >= 0; j--) {                 // j-th newest lives in slot (TT-1+u-j) mod TT
                    const float2 v = w[(2 * TT - 1 + u - j) % TT];
                    re = fmaf(v.x, tr[j], re); im = fmaf(v.y, tr[j], im);
                }
                fftbuf[(o + u) * N + b] = make_float2(re, im);
                w[u] = q[u];                                       // overwrite the oldest (slot u) with the next push
            }
        }
#pragma unroll
        for (int u = 0; u < TT; u++) q[u] = qn[u];
    }
}

// One thread per window b, walking a run of consecutive output vectors: everything that depends on the
// output index (newest push of the window, how many of its T samples come from this call, which arm the
// window meets) is advanced with adds and compares instead of the six 64-bit divisions per output the
// first version spent -- they, not the 2*T FMAs, were the cost of this kernel.  Loads are coalesced across
// b (adjacent windows receive adjacent input samples); the T-sample reuse between consecutive outputs of a
// thread is served by L1.  The MAC order is the reference's (oldest sample first, channelizer.rs:186-199).
__global__ void chan_bank_kernel(const float2 *__restrict__ in, const float2 *__restrict__ hist,
                                 const float *__restrict__ arms, float2 *__restrict__ fftbuf, int N, int D, int T,
                                 int base0, long long nprod, int orun) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;               // window / fft_buf index
    if (b >= N) return;
    const long long o_begin = (long long)blockIdx.y * orun;
    const long long o_end = min(o_begin + (long long)orun, nprod);
    if (o_begin >= o_end) return;
    const int r = ((base0 - b) % N + N) % N;                           // this window receives pushes c == r (mod N)
    // closed forms at the first output of the run
    long long E = (o_begin + 1) * D;                                   // pushes done when output o is formed
    long long c_new = -1; int m = 0;
    if (E - 1 >= r) { c_new = r + ((E - 1 - r) / N) * N; m = (int)((c_new - r) / N) + 1; }
    int base_after = (int)(((base0 - E) % N + N) % N);
    const float2 *hb = hist + (size_t)b * T;
    if (D == N && m >= T) {
        int i = b - base_after - 1;
        if (i < 0) i += N;
        switch (T) {
            case 4: chan_run_regs<4>(in, arms + i, fftbuf, N, b, c_new, o_begin, o_end); return;
            case 8: chan_run_regs<8>(in, arms + i, fftbuf, N, b, c_new, o_begin, o_end); return;
            case 16: chan_run_regs<16>(in, arms + i, fftbuf, N, b, c_new, o_begin, o_end); return;
            default: break;
        }
    }
    for (long long o = o_begin; o < o_end; o++) {
        int i = b - base_after - 1;                                    // arm: b = (base_after + i + 1) % N
        if (i < 0) i += N;
        const float *a = arms + i;                                     // arm i, tap j at a[j * N]
        float re = 0.f, im = 0.f;
        // reference order: t = 0 (oldest) .. T-1 with tap arm[T-1-t]  <=>  j = T-1 .. 0 with tap arm[j]
        if (m >= T) {                                                  // steady state: all T samples are in this call's input
            const float2 *xp = in + (c_new - (long long)(T - 1) * N);    // oldest sample first
            const float *ap = a + (size_t)(T - 1) * N;
#pragma unroll 4
            for (int j = 0; j < T; j++, xp += N, ap -= N) {
                const float2 v = __ldg(xp);
                const float tap = __ldg(ap);
                re = fmaf(v.x, tap, re); im = fmaf(v.y, tap, im);
            }
        } else {
            for (int j = T - 1; j >= 0; j--) {
                const float2 v = (j < m) ? __ldg(in + (c_new - (long long)j * N)) : hb[T - 1 - (j - m)];
                const float tap = __ldg(a + (size_t)j * N);
                re = fmaf(v.x, tap, re); im = fmaf(v.y, tap, im);
            }
        }
        fftbuf[o * N + b] = make_float2(re, im);
        // advance to output o + 1:  E += D (D <= N, so the window gains at most one sample)
        E += D;
        if (c_new < 0) { if (E - 1 >= r) { c_new = r; m = 1; } }
        else if (c_new + N <= E - 1) { c_new += N; m++; }
        base_after -= D;
        if (base_after < 0) base_after += N;
    }
}

__global__ void chan_hist_update(float2 *hist, const float2 *__restrict__ in, int N, int T, int base0, long long npush) {
    extern __shared__ float2 tmp[];
    const int b = blockIdx.x;
    const int r = ((base0 - b) % N + N) % N;
    long long c_new = -1; int m = 0;
    if (npush - 1 >= r) { c_new = r + ((npush - 1 - r) / N) * N; m = (int)((c_new - r) / N) + 1; }
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const int j = T - 1 - t;                                       // new hist[t] = j-th newest
        tmp[t] = (j < m) ? in[c_new - (long long)j * N] : hist[(size_t)b * T + (T - 1 - (j - m))];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) hist[(size_t)b * T + t] = tmp[t];
}

// out[ch * stride + o] = spec[o * N + ch]
__global__ void chan_transpose_kernel(const float2 *__restrict__ spec, float2 *__restrict__ out, int N, long long nprod,
                                      long long stride) {
    __shared__ float2 tile[32][33];
    const long long o0 = (long long)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const long long o = o0 + i; const int ch = c0 + threadIdx.x;
        if (o < nprod && ch < N) tile[i][threadIdx.x] = spec[o * N + ch];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int ch = c0 + i; const long long o = o0 + threadIdx.x;
        if (o < nprod && ch < N) out[(long long)ch * stride + o] = tile[threadIdx.x][i];
    }
}

// ---------------------------------------------------------------------------------------------------------------
// FUSED steady state (critically sampled, N a power of two <= 256, T <= 32): FIR bank + N-point inverse FFT +
// channel-major store in ONE kernel -- 8 B/sample in, 8 B/sample out, nothing in between touches HBM (the three
// kernels above move 48 B/sample).  A CTA owns OB consecutive output vectors:
//   A. the (OB + TPAD - 1) * N input samples they depend on are copied to shared memory (one contiguous span:
//      window b receives the samples congruent to r_b mod N, so row q of the tile is in[q*N .. q*N+N));
//   B. thread (window b, run of RL consecutive outputs) streams its column of the tile through registers ONCE:
//      every loaded sample is multiplied into all outputs of the run that contain it (taps in registers, static
//      indices after unrolling) -- 1 LDS.64 per ~RL*TPAD/(RL+TPAD-1) complex MACs, MAC order oldest sample first
//      exactly like channelizer.rs:186-199;
//   C. the OB vectors are de-spun by the Stockham passes of fft_common.cuh in shared memory (inverse = conj o FFT o conj);
//   D. results leave transposed: for each channel the OB outputs are contiguous in its output stream.
// Outputs whose windows still reach into the previous call's history (the first T-1 of a call) take the generic
// three-kernel path.
// ---------------------------------------------------------------------------------------------------------------
// Row stride of the FFT buffers = the padded transform length fft_geom(..).np.  (The exact, odd stride N + N/16 - 1
// puts the 512/N transforms a warp works on at distinct bank offsets, but its rows start 8 bytes off a 16-byte
// boundary, which cost more than the bank conflicts it removes.  Also: at 68 the 64-channel kernel sits at EXACTLY two
// CTAs per SM, 2 x (2 x 40448 + 64 x 68 x 8 + 1024 reserved) = 233472 bytes; one float2 more per row halves the
// occupancy.)

// items of one input tile: (OB + TPAD - 1) x N samples, reused as the transposed [OB][N+1] output staging
constexpr size_t chan_xcap(int log2n, int tpad) {
    const fftk::FftGeom g = fftk::fft_geom(log2n, 256);
    const size_t rows = (size_t)(g.fpb + tpad - 1) * g.n, staging = (size_t)g.fpb * (g.n + 1);
    return rows > staging ? rows : staging;
}

__device__ __forceinline__ void chan_cp_async16(void *dst_smem, const void *src, bool valid) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
    const int sz = valid ? 16 : 0;                       // src-size 0: the 16 bytes are zero-filled
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}

// Persistent: a CTA walks tiles blockIdx.x, blockIdx.x + gridDim.x, ... and the input tile of the NEXT one is fetched
// with cp.async into the other half of a double buffer while the current one is filtered, transformed and stored
// (a load, wait, compute sequence leaves the CTA stalled on its global loads).
template <int LOG2N, int TPAD>
__global__ void __launch_bounds__(256) chan_fused_kernel(const float2 *__restrict__ in, const float *__restrict__ arms_pad,
                                                         const float2 *__restrict__ tw, float2 *__restrict__ out, int base0,
                                                         long long o_first, long long nprod, long long out_stride, int ntiles) {
    using namespace fftk;
    constexpr FftGeom G = fft_geom(LOG2N, 256);
    constexpr int N = G.n, TT = G.t, NP = G.np;              // TT threads per transform
    constexpr int OB = G.fpb;                                // output vectors per tile
    constexpr int RUNS = 256 / N;                            // runs of outputs per window
    constexpr int RL = OB / RUNS;                            // outputs per run
    constexpr int ROWS = OB + TPAD - 1;
    constexpr size_t XCAP = chan_xcap(LOG2N, TPAD);
    extern __shared__ __align__(16) unsigned char csm[];
    float2 *Xbuf = reinterpret_cast<float2 *>(csm);          // 2 x [ROWS][N] input tiles (each reused as the transposed staging [OB][N+1])
    float2 *V = Xbuf + 2 * XCAP;                             // [OB][NP]    FFT buffers
    const int tid = threadIdx.x;
    const long long n_items = nprod * N;

    // window geometry and taps of this thread: the same for every tile (critically sampled)
    const int b = tid % N, run = tid / N;
    int r = (base0 - b) % N; if (r < 0) r += N;              // window b receives samples == r (mod N)
    int arm = (b - base0 - 1) % N; if (arm < 0) arm += N;    // and always meets this arm
    float tap[TPAD];
#pragma unroll
    for (int j = 0; j < TPAD; j++) tap[j] = __ldg(arms_pad + (size_t)j * N + arm);

    auto fetch = [&](int tile, float2 *X) {                  // A: the (OB + TPAD - 1) * N samples tile `tile` depends on
        const long long base = (o_first + (long long)tile * OB - (TPAD - 1)) * N;   // rows in front of the call meet zero taps
        constexpr int TOT4 = ROWS * N / 2;                   // 16 bytes = 2 samples
        for (int e = tid; e < TOT4; e += 256) {
            const long long it = base + 2ll * e;             // even, and n_items is even: both samples valid or none
            const bool ok = it >= 0 && it + 1 < n_items;
            chan_cp_async16(reinterpret_cast<float4 *>(X) + e, in + (ok ? it : 0), ok);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    int it_n = 0;
    if ((int)blockIdx.x < ntiles) fetch(blockIdx.x, Xbuf);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, it_n++) {
        float2 *X = Xbuf + (size_t)(it_n & 1) * XCAP;
        const int nxt = tile + gridDim.x;
        if (nxt < ntiles) {
            fetch(nxt, Xbuf + (size_t)((it_n & 1) ^ 1) * XCAP);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        const long long o0 = o_first + (long long)tile * OB;

        // ---- B: FIR bank (every sample of the column is loaded once and multiplied into all outputs that contain it)
        {
            float2 acc[RL];
#pragma unroll
            for (int u = 0; u < RL; u++) acc[u] = make_float2(0.f, 0.f);
            const float2 *col = X + (size_t)(run * RL) * N + r;   // tile row (run*RL + k) <-> sample row o_run - TPAD + 1 + k
#pragma unroll
            for (int k = 0; k < RL + TPAD - 1; k++) {
                const float2 x = col[(size_t)k * N];
#pragma unroll
                for (int u = 0; u < RL; u++) {
                    const int j = u + TPAD - 1 - k;          // output u sees this row as its j-th newest sample
                    if (j >= 0 && j < TPAD) mac(acc[u], x, tap[j]);
                }
            }
#pragma unroll
            for (int u = 0; u < RL; u++)                      // conjugated: the inverse transform is conj(FFT(conj(.)))
                V[(size_t)(run * RL + u) * NP + pad(b)] = make_float2(acc[u].x, -acc[u].y);
        }
        __syncthreads();

        // ---- C: N-point FFT of every vector; conjugate + transposed staging in the (now free) tile
        {
            const int ol = tid / TT, t = tid % TT;
            float2 *sm = V + (size_t)ol * NP;
            fft_passes<LOG2N, TT, Tw::Ahead>([&](int idx) { return sm[pad(idx)]; },
                                             [&](int idx, float2 v) { X[(size_t)ol * (N + 1) + idx] = make_float2(v.x, -v.y); },
                                             sm, tw, t, true);
        }
        // (fft_passes ends with a CTA barrier)  ---- D: for each channel the OB outputs are contiguous
        for (int e = tid; e < OB * N; e += 256) {
            const int ch = e / OB, ol = e % OB;
            if (o0 + ol < nprod) out[(long long)ch * out_stride + o0 + ol] = X[(size_t)ol * (N + 1) + ch];
        }
        __syncthreads();                                      // X is the next iteration's prefetch target
    }
}

template <int LOG2N, int TPAD> constexpr size_t chan_fused_smem() {
    constexpr fftk::FftGeom G = fftk::fft_geom(LOG2N, 256);
    return (2 * chan_xcap(LOG2N, TPAD) + (size_t)G.fpb * G.np) * sizeof(float2);
}

static inline bool ntiles_overflow(long long nprod, long long o_first, int ob) { return (nprod - o_first) / ob > 0x7fffff00ll; }

template <int LOG2N, int TPAD>
int32_t chan_fused_launch(b2s_chan *c, const float2 *in, float2 *out, long long o_first, long long nprod, long long out_stride) {
    constexpr int OB = fftk::fft_geom(LOG2N, 256).fpb;
    constexpr size_t smem = chan_fused_smem<LOG2N, TPAD>();
    auto kern = chan_fused_kernel<LOG2N, TPAD>;
    static PerDeviceOnce optin;
    if (ntiles_overflow(nprod, o_first, OB)) return b2s_fail(c->ctx, B2S_EUNSUPPORTED, "channelizer: too many output vectors in one call");
    if (smem > 48 * 1024 && optin.need(c->ctx->device)) {
        B2S_CUDA(c->ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        optin.done(c->ctx->device);
    }
    const size_t ntiles = ceil_div((size_t)(nprod - o_first), (size_t)OB);
    static int resident = 0;                                  // CTAs per SM of this instantiation
    if (!resident) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, 256, smem) != cudaSuccess || resident < 1) { cudaGetLastError(); resident = 1; }
    }
    const unsigned grid = (unsigned)std::min<size_t>(ntiles, (size_t)c->ctx->sm_count * resident);
    kern<<<grid, 256, smem, c->ctx->stream>>>(in, c->d_arms_pad.get(), b2s_fft_twiddles(c->ifft.get()), out, (int)c->base_index, o_first,
                                             nprod, out_stride, (int)ntiles);
    B2S_CHECK_LAUNCH(c->ctx);
    return B2S_OK;
}

template <int TPAD>
int32_t chan_fused_dispatch(b2s_chan *c, int log2n, const float2 *in, float2 *out, long long o_first, long long nprod,
                            long long out_stride) {
    return fftk::with_log2n<2, 8>(log2n, B2S_EAGAIN,
                                  [&](auto L) { return chan_fused_launch<L, TPAD>(c, in, out, o_first, nprod, out_stride); });
}

// TPAD (8 / 16 / 32) the fused kernel would use for this plan, 0 if the plan is outside its shapes
int chan_fused_tpad(const b2s_chan *c) {
    const int l2 = b2s_fft_log2n(c->ifft.get());
    if (getenv("B2S_CHAN_NO_FUSED")) return 0;
    if (l2 < 2 || l2 > 8 || c->D != c->N || c->T > 32) return 0;
    return c->T <= 8 ? 8 : (c->T <= 16 ? 16 : 32);
}

}  // namespace

extern "C" {

int32_t b2s_chan_plan_c32(b2s_ctx *ctx, size_t num_channels, const float *taps, size_t ntaps, float oversample_rate,
                          b2s_chan **out) {
    if (!ctx || !out || !taps) return b2s_fail(ctx, B2S_EINVAL, "b2s_chan_plan_c32: NULL argument");
    *out = nullptr;
    // the reference asserts these (channelizer.rs:92-104)
    if (num_channels <= 2) return b2s_fail(ctx, B2S_EINVAL, "PfbChannelizer: number of channels must be at least 2");
    if (ntaps < num_channels) return b2s_fail(ctx, B2S_EINVAL, "PfbChannelizer: prototype filter length must be at least num_channels");
    if (oversample_rate == 0.f || std::fmod((float)num_channels, oversample_rate) != 0.f)
        return b2s_fail(ctx, B2S_EINVAL, "pfb_channelizer: oversample rate must be N/i for i in [1, N]");
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_chan> c(new b2s_chan());
    c->ctx = ctx; c->N = num_channels;
    c->D = (size_t)((float)num_channels / oversample_rate);                      // channelizer.rs:106
    const size_t N = c->N, T = (size_t)std::ceil((float)ntaps / (float)N);       // utilities.rs:9
    c->T = T;
    std::vector<float> arms(N * T, 0.0f);
    for (size_t i = 0; i < N; i++) { size_t j = 0; for (size_t idx = i; idx < ntaps; idx += N) arms[(j++) * N + i] = taps[idx]; }
    c->start_idx.assign(N, 0); c->missing.assign(N, (int)T);
    c->base_index = N - 1;
    b2s_fft *ifft = nullptr;
    B2S_TRY(b2s_fft_plan_c32(ctx, N, 1, 0, 0, 1.0f, &ifft));                    // plan_fft(n, Inverse) (:114)
    c->ifft.reset(ifft);
    std::vector<int> ws(2 * N);
    for (size_t i = 0; i < N; i++) { ws[i] = 0; ws[N + i] = (int)T; }
    B2S_TRY(c->d_arms.upload(ctx, arms.data(), arms.size(), "channelizer arms"));
    B2S_TRY(c->d_circ.alloc(ctx, N * 2 * T, "channelizer windows"));
    B2S_TRY(c->d_hist.alloc(ctx, N * T, "channelizer history"));
    B2S_TRY(c->d_wstate.upload(ctx, ws.data(), ws.size(), "channelizer window state"));
    B2S_CUDA(ctx, cudaMemsetAsync(c->d_circ.get(), 0, N * 2 * T * sizeof(float2), ctx->stream));
    c->tpad = chan_fused_tpad(c.get());
    std::vector<float> apad;
    if (c->tpad) {
        apad.assign((size_t)c->tpad * N, 0.0f);                                  // taps beyond T are zero (older samples)
        std::copy(arms.begin(), arms.end(), apad.begin());
        B2S_TRY(c->d_arms_pad.upload(ctx, apad.data(), apad.size(), "channelizer padded arms"));
    }
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *out = c.release();
    return B2S_OK;
}

void b2s_chan_destroy(b2s_chan *c) { PlanDeleter<b2s_chan>()(c); }

size_t b2s_chan_decimation(const b2s_chan *c) { return c ? c->D : 0; }

// One Kernel::work call (channelizer.rs:142-223).  d_out is channel-major: stream ch starts at
// d_out + ch * out_stride items; n_out_cap = the smallest free space over the N output slices.
int32_t b2s_chan_exec(b2s_chan *c, const void *d_in, size_t n_in, void *d_out, size_t out_stride, size_t n_out_cap,
                      size_t *consumed, size_t *produced_per_channel, int32_t *call_again) {
    if (!c || !consumed || !produced_per_channel || !call_again)
        return b2s_fail(c ? c->ctx : nullptr, B2S_EINVAL, "b2s_chan_exec: NULL argument");
    b2s_ctx *ctx = c->ctx;
    *consumed = 0; *produced_per_channel = 0; *call_again = 0;
    DeviceGuard g(ctx->device);
    const int N = (int)c->N, T = (int)c->T, D = (int)c->D;
    const float2 *in = (const float2 *)d_in;
    if (!c->all_filled) {
        // host mirror of the push bookkeeping decides how many samples this call pushes
        size_t cnt = 0;
        size_t base = c->base_index;
        auto all_filled = [&]() { for (int m : c->missing) if (m) return false; return true; };
        while (!all_filled() && cnt < n_in) {
            if (c->missing[base] > 0) c->missing[base]--;
            c->start_idx[base] = (c->start_idx[base] + 1) % T;
            base = base == 0 ? (size_t)N - 1 : base - 1;
            cnt++;
        }
        if (cnt) {
            if (!d_in) return b2s_fail(ctx, B2S_EINVAL, "b2s_chan_exec: NULL buffer");
            chan_fill_kernel<<<1, 32, 0, ctx->stream>>>(in, c->d_circ.get(), c->d_wstate.get(), N, T, (int)c->base_index, (int)cnt);
            B2S_CHECK_LAUNCH(ctx);
        }
        c->base_index = base;
        if (!all_filled()) { *consumed = cnt; return B2S_OK; }               // input exhausted first (:165-170)
        c->all_filled = true;
        chan_hist_from_circ<<<N, 64, 0, ctx->stream>>>(c->d_circ.get(), c->d_wstate.get(), c->d_hist.get(), N, T);
        B2S_CHECK_LAUNCH(ctx);
        if (n_in >= (size_t)D) *call_again = 1;                                // :176-177; NB nothing is consumed here
        return B2S_OK;
    }
    size_t nprod = n_in / D;
    if (nprod > n_out_cap) nprod = n_out_cap;                                  // :155-158
    if (nprod == 0) return B2S_OK;
    if (!d_in || !d_out) return b2s_fail(ctx, B2S_EINVAL, "b2s_chan_exec: NULL buffer");
    // the first T-1 output vectors of a call still reach into the previous call's history: generic path; the rest
    // (windows entirely inside this call's input) go through the fused kernel
    const bool fused_ok = c->tpad && (reinterpret_cast<uintptr_t>(d_in) & 15) == 0;      // the tile copy uses 16-byte loads
    const size_t n_generic = fused_ok ? std::min<size_t>(nprod, (size_t)T - 1) : nprod;
    NvtxRange nvtx("b2s_chan_exec");
    if (n_generic < nprod) {
        int32_t rc = B2S_EAGAIN;
        const int l2 = b2s_fft_log2n(c->ifft.get());
        if (c->tpad == 8) rc = chan_fused_dispatch<8>(c, l2, in, (float2 *)d_out, (long long)n_generic, (long long)nprod, (long long)out_stride);
        else if (c->tpad == 16) rc = chan_fused_dispatch<16>(c, l2, in, (float2 *)d_out, (long long)n_generic, (long long)nprod, (long long)out_stride);
        else if (c->tpad == 32) rc = chan_fused_dispatch<32>(c, l2, in, (float2 *)d_out, (long long)n_generic, (long long)nprod, (long long)out_stride);
        if (rc != B2S_OK) return rc == B2S_EAGAIN ? b2s_fail(ctx, B2S_ESTATE, "channelizer: fused shape mismatch") : rc;
    }
    const size_t nprod_all = nprod;
    nprod = n_generic;
    const size_t items = nprod * N;
    if (items && c->d_tmp.size() < 2 * items)
        B2S_TRY(c->d_tmp.reserve(ctx, 2 * (items * 5 / 4 + 1024), "channelizer workspace"));
    float2 *bank = c->d_tmp.get(), *spec = c->d_tmp.get() + c->d_tmp.size() / 2;
    if (items) {
    {
        const int th = (int)std::min<size_t>(128, round_up(N, 32));
        const unsigned gx = (unsigned)ceil_div(N, (size_t)th);
        // runs of outputs per thread: enough CTAs to fill the machine (~16 per SM), at least 32 outputs per run
        const size_t want_y = std::max<size_t>(1, (size_t)ctx->sm_count * 16 / gx);
        const size_t orun = std::max<size_t>(32, ceil_div(nprod, want_y));
        dim3 grid(gx, (unsigned)ceil_div(nprod, orun));
        chan_bank_kernel<<<grid, th, 0, ctx->stream>>>(in, c->d_hist.get(), c->d_arms.get(), bank, N, D, T, (int)c->base_index,
                                                       (long long)nprod, (int)orun);
    }
    B2S_CHECK_LAUNCH(ctx);
    size_t fc = 0, fp = 0;
    int32_t rc = b2s_fft_exec(c->ifft.get(), bank, items, spec, items, &fc, &fp);
    if (rc != B2S_OK) return rc;
    dim3 tg((unsigned)ceil_div(nprod, (size_t)32), (unsigned)ceil_div((size_t)N, (size_t)32));
    chan_transpose_kernel<<<tg, dim3(32, 8), 0, ctx->stream>>>(spec, (float2 *)d_out, N, (long long)nprod, (long long)out_stride);
    B2S_CHECK_LAUNCH(ctx);
    }
    nprod = nprod_all;
    const long long npush = (long long)nprod * D;
    chan_hist_update<<<N, 64, T * sizeof(float2), ctx->stream>>>(c->d_hist.get(), in, N, T, (int)c->base_index, npush);
    B2S_CHECK_LAUNCH(ctx);
    c->base_index = (size_t)((((long long)c->base_index - npush) % N + N) % N);
    *consumed = (size_t)npush; *produced_per_channel = nprod;
    return B2S_OK;
}

}  // extern "C"
