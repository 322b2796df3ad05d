// fir_f64.cu -- the f64 x f64 Filter impls (crates/futuredsp/src/fir.rs:217-226, decimating_fir.rs:117-130):
//     o[k] = sum_t i[D-1 + k*D + t] * taps[N-1-t]      accumulated in tap order, `accum + sample * tap`
// The GPU has little FP64 throughput and no SDR graph of the reference runs its hot path in f64 (the impl exists for
// the known-answer tests, fir.rs:343-365), so this is the plain form: one thread per output, taps in shared memory,
// UN-FUSED multiply and add in the reference's order -- bit-identical to the stable-Rust loop.
#include "fir.cuh"

namespace {
constexpr int kF64Threads = 256;
constexpr int kF64TapsSmem = 4096;            // taps staged in shared memory up to this count

__global__ void __launch_bounds__(kF64Threads)
fir_f64_kernel(const double *__restrict__ in, double *__restrict__ out, const double *__restrict__ g /*reversed taps*/,
               int ntaps, long long decim, long long n_out, int taps_in_smem) {
    extern __shared__ double gs[];
    if (taps_in_smem) {
        for (int i = threadIdx.x; i < ntaps; i += kF64Threads) gs[i] = g[i];
        __syncthreads();
    }
    const double *gt = taps_in_smem ? gs : g;
    const long long stride = (long long)gridDim.x * kF64Threads;
    for (long long k = (long long)blockIdx.x * kF64Threads + threadIdx.x; k < n_out; k += stride) {
        const double *x = in + (decim - 1) + k * decim;
        double sum = 0.0;
        for (int t = 0; t < ntaps; t++) sum = __dadd_rn(sum, __dmul_rn(x[t], gt[t]));
        out[k] = sum;
    }
}
}  // namespace

int32_t fir_f64_prepare(b2s_fir *f, const double *taps) {
    b2s_ctx *ctx = f->ctx;
    std::vector<double> g(f->ntaps);
    for (size_t t = 0; t < f->ntaps; t++) g[t] = taps[f->ntaps - 1 - t];
    B2S_TRY(f->d_taps64.upload(ctx, g.data(), g.size(), "f64 taps"));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B2S_OK;
}

int32_t fir_f64_launch(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out, cudaStream_t stream) {
    b2s_ctx *ctx = f->ctx;
    (void)n_in;
    if (n_out == 0) return B2S_OK;
    const int smem_taps = f->ntaps <= kF64TapsSmem;
    const unsigned grid = (unsigned)std::min<size_t>(ceil_div(n_out, (size_t)kF64Threads), (size_t)ctx->sm_count * 16);
    fir_f64_kernel<<<grid, kF64Threads, smem_taps ? f->ntaps * sizeof(double) : 0, stream>>>(
        (const double *)d_in, (double *)d_out, f->d_taps64.get(), (int)f->ntaps, (long long)f->decim, (long long)n_out, smem_taps);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}
