// fir_fft.cu -- overlap-save FFT convolution for LONG filters (ntaps > 257) on Complex<f32>
// streams, real or complex taps, no decimation.
//
// Same result as crates/futuredsp/src/fir.rs:77-88,  o[k] = sum_t i[k+t] * taps[N-1-t], evaluated
// per block of NF = 4096 inputs as  y = IFFT( FFT(x_block) . H ),  H[f] = (1/NF) sum_t g[t]
// e^{+2 pi i f t / NF}  (g[t] = taps[N-1-t]; the correlation theorem), keeping the V = NF-(N-1)
// outputs that do not wrap.  One CTA owns one block: forward transform, spectrum product and
// inverse transform all happen in ONE kernel with the block resident in (padded) shared memory
// -- HBM sees 8 B in (x NF/V overlap, mostly L2 hits) + 8 B out per sample, instead of the
// 4*N FLOP per sample of the direct form (4096 FLOP/sample at 1024 taps).  Radix-16 Stockham passes from fft_common.cuh; H is computed in f64 on the host.
// Parity: the error follows the block's INPUT, not y: |err| <= 8 * 2^-24 * log2(NF) * (||taps||_2 * rms(x_block) +
// rms(circular output of the block)) -- a full-scale stopband tone gets an error near rms(y) -- and a NaN/Inf input
// poisons every output of each block that reads it (include/b200sdr.h, B2S_ALGO_FFT; tests/test_gpu_fir_fft_numerics.py).
// Most of the error is the Stockham core's product-tree twiddles (fft_common.cuh): about 3x what exact twiddles give.
#include <cmath>

#include "fft_common.cuh"
#include "fir.cuh"

using namespace fftk;

namespace {

constexpr int kLog2NF = 12;
constexpr int kNF = 1 << kLog2NF;
constexpr int kFfThreads = 256;

struct FftFirArgs {
    const float2 *in;
    float2 *out;
    const float2 *H;    // [NF]
    const float2 *tw;   // W_NF[k] = exp(-2 pi i k / NF)
    long long n_in, n_out;
    int V;              // valid outputs per block
};

// __launch_bounds__(256, 2): the unconstrained build takes ONE 256-thread CTA per SM by registers; a minimum of two
// CTAs per SM caps it at 128 registers.  (A template, with this one instantiation, so that profiles name it
// fir_fft_kernel<2>.)
template <int MINB>
__global__ void __launch_bounds__(kFfThreads, MINB) fir_fft_kernel(const FftFirArgs a) {
    extern __shared__ __align__(16) unsigned char ffsm[];
    float2 *sm = reinterpret_cast<float2 *>(ffsm);
    const int t = threadIdx.x;
    const long long s = (long long)blockIdx.x * a.V;
    const float2 *in = a.in + s;
    const long long avail = a.n_in - s;                 // items readable from `in`
    static_assert(fft_geom(kLog2NF, kFfThreads).t == kFfThreads, "one transform per CTA");

    // forward: global -> sm.  Every pass's base twiddle is fetched one pass ahead (Tw::Ahead).
    fft_passes<kLog2NF, kFfThreads, Tw::Ahead>([&](int idx) { return idx < avail ? __ldg(in + idx) : make_float2(0.f, 0.f); },
                                              [&](int idx, float2 v) { sm[pad(idx)] = v; }, sm, a.tw, t, false);
    // inverse = conj(FFT(conj(X . H))): spectrum product + conjugation fused into the first load, the final
    // conjugation into the store of the V valid outputs
    const long long room = a.n_out - s;
    float2 *out = a.out + s;
    const int V = a.V;
    fft_passes<kLog2NF, kFfThreads, Tw::Ahead>(
        [&](int idx) {
            const float2 y = cmul(sm[pad(idx)], __ldg(a.H + idx));
            return make_float2(y.x, -y.y);
        },
        [&](int idx, float2 v) {
            if (idx < V && idx < room) out[idx] = make_float2(v.x, -v.y);
        },
        sm, a.tw, t, true);
}

}  // namespace

bool fir_fft_supported(const b2s_fir *f) {
    if (f->decim != 1) return false;
    if (f->kind != B2S_C32_F32 && f->kind != B2S_C32_C32) return false;
    return f->ntaps >= 64 && f->ntaps <= kNF / 2 + 1;      // V >= NF/2
}

int32_t fir_fft_prepare(b2s_fir *f) {
    b2s_ctx *ctx = f->ctx;
    if (f->d_fftH) return B2S_OK;
    if (!fir_fft_supported(f)) return b2s_fail(ctx, B2S_EUNSUPPORTED, "FFT FIR: unsupported plan");
    const size_t N = f->ntaps;
    const bool ctap = f->kind == B2S_C32_C32;
    const double PI = 3.14159265358979323846264338327950288;
    std::vector<float2> H(kNF);
    // H[f] = (1/NF) sum_t g[t] e^{+2 pi i f t / NF},  g[t] = taps[N-1-t]
    std::vector<double> cs(kNF), sn(kNF);
    for (int k = 0; k < kNF; k++) {
        const double ang = 2.0 * PI * (double)k / (double)kNF;
        cs[k] = std::cos(ang); sn[k] = std::sin(ang);
    }
    for (int fr = 0; fr < kNF; fr++) {
        double re = 0.0, im = 0.0;
        for (size_t t = 0; t < N; t++) {
            const size_t src = N - 1 - t;
            const double gr = ctap ? f->taps_host[2 * src] : f->taps_host[src];
            const double gi = ctap ? f->taps_host[2 * src + 1] : 0.0;
            const int k = (int)(((size_t)fr * t) & (kNF - 1));
            re += gr * cs[k] - gi * sn[k];
            im += gr * sn[k] + gi * cs[k];
        }
        H[fr] = make_float2((float)(re / kNF), (float)(im / kNF));
    }
    const std::vector<float2> tw = twiddle_table(kNF);
    H.insert(H.end(), tw.begin(), tw.end());
    B2S_TRY(f->d_fftH.upload(ctx, H.data(), H.size(), "FFT FIR spectrum"));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B2S_OK;
}

int32_t fir_fft_launch(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out, cudaStream_t stream) {
    b2s_ctx *ctx = f->ctx;
    if (n_out == 0) return B2S_OK;
    if (!f->d_fftH) return b2s_fail(ctx, B2S_ESTATE, "FFT FIR not prepared");
    if ((reinterpret_cast<uintptr_t>(d_in) | reinterpret_cast<uintptr_t>(d_out)) & 7)
        return fir_direct_launch(f, d_in, n_in, d_out, n_out, stream);
    FftFirArgs a;
    a.in = (const float2 *)d_in; a.out = (float2 *)d_out;
    a.H = f->d_fftH.get(); a.tw = f->d_fftH.get() + kNF;
    a.n_in = (long long)n_in; a.n_out = (long long)n_out;
    a.V = kNF - (int)(f->ntaps - 1);
    const unsigned grid = (unsigned)ceil_div(n_out, (size_t)a.V);
    const size_t smem = (size_t)fft_geom(kLog2NF, kFfThreads).np * sizeof(float2);
    fir_fft_kernel<2><<<grid, kFfThreads, smem, stream>>>(a);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}
