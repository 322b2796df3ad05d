// fir.cuh -- FIR plan object shared by the ABI layer and the kernel translation units.
#pragma once
#include "common.cuh"

struct b2s_fir {
    b2s_ctx *ctx = nullptr;
    b2s_kind kind = B2S_C32_F32;
    size_t ntaps = 0, decim = 1;
    std::vector<float> taps_host;   // reference order, kind_tap_floats(kind) floats per tap
    b2s_algo algo_req = B2S_ALGO_AUTO, algo = B2S_ALGO_DIRECT;

    // ---- direct form (fir_direct.cu): per-phase, time-reversed, zero-padded taps in HBM.
    // G[q][u] = g[D*u + q - (D-1)] (u < Upad), then g[t] = taps[N-1-t]   (see DESIGN.md "direct FIR")
    Buf<float> d_ptaps;
    int Upad = 0;

    // ---- tensor-core form (fir_tc.cu): split-bf16 Toeplitz blocks, built lazily
    int tc_kblocks = 0;
    bool tc_ready = false;
    int tc_flags = 0;            // bring-up switches (env B2S_TC_FLAGS)
    Buf<unsigned> d_tc_sched;    // per-launch tile counters {next tile, CTAs done}, zero between launches
    unsigned tc_launches = 0;

    // ---- FFT overlap-save form (fir_fft.cu): H[NF] then W_NF[NF], built lazily
    Buf<float2> d_fftH;

    // ---- f64 x f64 (fir_f64.cu): reversed taps in double precision
    Buf<double> d_taps64;
};

// fir_direct.cu
int32_t fir_direct_prepare(b2s_fir *f);
int32_t fir_direct_launch(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out,
                          cudaStream_t stream);
// fir_direct.cu: rational resampler on the same kernel (called from resamp.cu)
std::vector<float> slide_table(const float *taps, size_t tf, size_t L, size_t M, size_t T, size_t lead);
bool    resamp_slide_supported(size_t L, size_t M, size_t T, size_t item_bytes);
int32_t resamp_slide_launch(b2s_ctx *ctx, b2s_kind kind, const float *d_gtab, size_t L, size_t M, size_t T,
                            const void *d_in, size_t n_in, void *d_out, size_t n_out, cudaStream_t stream);
// detached history of b2s_fir_exec_hist: n_hist items that logically precede the slice, plus the optional
// cross-GPU handshake (system-scope flags in device memory, see peer.cu)
struct FirHist {
    const void *d_hist = nullptr;
    size_t n_hist = 0;
    unsigned *publish_flag = nullptr;
    unsigned publish_value = 0;
    const unsigned *wait_flag = nullptr;
    unsigned wait_value = 0;
    unsigned *done_flag = nullptr;
    unsigned done_value = 0;
};
// fir_tc.cu
bool    fir_tc_supported(const b2s_fir *f);
int32_t fir_tc_launch_hist(b2s_fir *f, const FirHist *h, const void *d_in, size_t n_in, void *d_out, size_t n_out,
                           cudaStream_t stream);
int32_t fir_tc_prepare(b2s_fir *f);
int32_t fir_tc_launch(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out,
                      cudaStream_t stream);
// fir_f64.cu
int32_t fir_f64_prepare(b2s_fir *f, const double *taps);
int32_t fir_f64_launch(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out, cudaStream_t stream);
// fir_fft.cu
bool    fir_fft_supported(const b2s_fir *f);
int32_t fir_fft_prepare(b2s_fir *f);
int32_t fir_fft_launch(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out,
                       cudaStream_t stream);
