// chan.cu -- polyphase channelizer (src/blocks/pfb/channelizer.rs:88-223) on the device:
// SURVEY.md §8f row 2, a pure composition of the FIR-bank and FFT pieces of the hot path.
//
// Reference semantics restated: every consumed sample is pushed into window `base_index`, which
// then decrements modulo N -- so window w holds the stream decimated by N at phase (base0 - w);
// after each group of D = N / oversample_rate pushes, arm i (taps[i::N]) filters window
// (base_index + i + 1) % N into fft_buf[that window], an un-normalised inverse FFT over the N
// buffers de-spins, and element ch goes to output stream ch.
//   * start-up: the windows fill through the shared window buffer of pfb_common.cuh (sample c of the
//     stream goes to window N-1 - c mod N), and the call in which the last window fills returns
//     WITHOUT consuming (channelizer.rs:170-180), so those samples are pushed a second time.
//   * steady state is closed-form: one thread per (output vector o, window b) gathers the T newest
//     samples of its phase (history buffer + this call's input) and dots them with its arm; the
//     N-point inverse FFT is the batched FFT kernel of fft.cu (any N: radix or Bluestein), a
//     transposing store writes channel-major output streams.
#include <cstdlib>

#include "pfb_common.cuh"

struct b2s_chan {
    b2s_ctx *ctx = nullptr;
    size_t N = 0, D = 0, T = 0;
    PfbBankTaps taps;               // arm i meets window (base_index + i + 1) % N
    PfbWindows win;                 // N windows, mirrored: window base_index receives the next sample
    size_t base_index = 0;
    PlanPtr<b2s_fft> ifft;
    Buf<float2> d_tmp;              // two halves: bank outputs, spectra
};

namespace {

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

// Persistent: a CTA walks tiles blockIdx.x, blockIdx.x + gridDim.x, ... and the input tile of the NEXT one is fetched
// with cp.async into the other half of a double buffer while the current one is filtered, transformed and stored
// (a load, wait, compute sequence leaves the CTA stalled on its global loads).
template <int LOG2N, int TPAD, bool PADDED>
__global__ void __launch_bounds__(256) chan_fused_kernel(const float2 *__restrict__ in, const float *__restrict__ arms_pad,
                                                         const float2 *__restrict__ tw, float2 *__restrict__ out, int T,
                                                         int base0, long long o_first, long long nprod, long long out_stride,
                                                         int ntiles) {
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
            cp_async::cg16(reinterpret_cast<float4 *>(X) + e, in + (ok ? it : 0), ok);
        }
        cp_async::commit();
    };

    int it_n = 0;
    if ((int)blockIdx.x < ntiles) fetch(blockIdx.x, Xbuf);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, it_n++) {
        float2 *X = Xbuf + (size_t)(it_n & 1) * XCAP;
        const int nxt = tile + gridDim.x;
        if (nxt < ntiles) {
            fetch(nxt, Xbuf + (size_t)((it_n & 1) ^ 1) * XCAP);
            cp_async::wait<1>();
        } else {
            cp_async::wait<0>();
        }
        __syncthreads();
        const long long o0 = o_first + (long long)tile * OB;

        // ---- B: FIR bank (every sample of the column is loaded once and multiplied into all outputs that contain it)
        {
            float2 acc[RL];
            // tile row (run*RL + k) <-> sample row o_run - TPAD + 1 + k
            pfb_bank_column<N, RL, TPAD, PADDED>(X + (size_t)(run * RL) * N + r, tap, T, acc);
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

template <int LOG2N, int TPAD, bool PADDED>
int32_t chan_fused_launch(b2s_chan *c, const float2 *in, float2 *out, long long o_first, long long nprod, long long out_stride) {
    constexpr int OB = fftk::fft_geom(LOG2N, 256).fpb;
    constexpr size_t smem = chan_fused_smem<LOG2N, TPAD>();
    if (ntiles_overflow(nprod, o_first, OB)) return b2s_fail(c->ctx, B2S_EUNSUPPORTED, "channelizer: too many output vectors in one call");
    constexpr auto kern = chan_fused_kernel<LOG2N, TPAD, PADDED>;
    int resident = 1;
    B2S_TRY(smem_optin<kern>(c->ctx, smem, 256, &resident));
    const size_t ntiles = ceil_div((size_t)(nprod - o_first), (size_t)OB);
    const unsigned grid = (unsigned)std::min<size_t>(ntiles, (size_t)c->ctx->sm_count * resident);
    kern<<<grid, 256, smem, c->ctx->stream>>>(in, c->taps.arms_pad.get(), b2s_fft_twiddles(c->ifft.get()), out, (int)c->T,
                                             (int)c->base_index, o_first, nprod, out_stride, (int)ntiles);
    B2S_CHECK_LAUNCH(c->ctx);
    return B2S_OK;
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
    const size_t N = c->N;
    std::vector<float> arms;
    const size_t T = pfb_partition(taps, ntaps, N, arms);
    c->T = T;
    c->base_index = N - 1;
    b2s_fft *ifft = nullptr;
    B2S_TRY(b2s_fft_plan_c32(ctx, N, 1, 0, 0, 1.0f, &ifft));                    // plan_fft(n, Inverse) (:114)
    c->ifft.reset(ifft);
    const int tpad = getenv("B2S_CHAN_NO_FUSED") || c->D != N ? 0 : pfb_fused_tpad(b2s_fft_log2n(ifft), T);
    B2S_TRY(c->taps.upload(ctx, arms, N, T, tpad, "channelizer arms"));
    B2S_TRY(c->win.init(ctx, (int)N, (int)T, true, "channelizer windows"));
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
    if (!c->win.full()) {
        const size_t cnt = std::min(n_in, c->win.missing());
        if (cnt && !d_in) return b2s_fail(ctx, B2S_EINVAL, "b2s_chan_exec: NULL buffer");
        B2S_TRY(c->win.push(ctx, in, cnt));
        c->base_index = (size_t)((((long long)c->base_index - (long long)cnt) % N + N) % N);
        if (!c->win.full()) { *consumed = cnt; return B2S_OK; }              // input exhausted first (:165-170)
        if (n_in >= (size_t)D) *call_again = 1;                                // :176-177; NB nothing is consumed here
        return B2S_OK;
    }
    size_t nprod = n_in / D;
    if (nprod > n_out_cap) nprod = n_out_cap;                                  // :155-158
    if (nprod == 0) return B2S_OK;
    if (!d_in || !d_out) return b2s_fail(ctx, B2S_EINVAL, "b2s_chan_exec: NULL buffer");
    // the first T-1 output vectors of a call still reach into the previous call's history: generic path; the rest
    // (windows entirely inside this call's input) go through the fused kernel
    const bool fused_ok = c->taps.tpad && (reinterpret_cast<uintptr_t>(d_in) & 15) == 0;      // the tile copy uses 16-byte loads
    const size_t n_generic = fused_ok ? std::min<size_t>(nprod, (size_t)T - 1) : nprod;
    NvtxRange nvtx("b2s_chan_exec");
    if (n_generic < nprod) {
        const int32_t rc = pfb_fused_dispatch(b2s_fft_log2n(c->ifft.get()), c->taps.tpad, c->T, [&](auto L, auto P, auto D) {
            return chan_fused_launch<L, P, D>(c, in, (float2 *)d_out, (long long)n_generic, (long long)nprod, (long long)out_stride);
        });
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
        chan_bank_kernel<<<grid, th, 0, ctx->stream>>>(in, c->win.hist.get(), c->taps.arms.get(), bank, N, D, T, (int)c->base_index,
                                                       (long long)nprod, (int)orun);
    }
    B2S_CHECK_LAUNCH(ctx);
    size_t fc = 0, fp = 0;
    int32_t rc = b2s_fft_exec(c->ifft.get(), bank, items, spec, items, &fc, &fp);
    if (rc != B2S_OK) return rc;
    B2S_TRY(pfb_transpose(ctx, spec, (float2 *)d_out, nprod, N, N, out_stride));   // out[ch * out_stride + o] = spec[o * N + ch]
    }
    nprod = nprod_all;
    const long long npush = (long long)nprod * D;
    B2S_TRY(c->win.slide(ctx, in, N - 1 - (long long)c->base_index, npush));   // sample 0 goes to window base_index
    c->base_index = (size_t)((((long long)c->base_index - npush) % N + N) % N);
    *consumed = (size_t)npush; *produced_per_channel = nprod;
    return B2S_OK;
}

}  // extern "C"
