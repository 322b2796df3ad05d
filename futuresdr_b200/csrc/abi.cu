// abi.cu -- context, memory and FIR entry points of the C ABI (include/b200sdr.h).
#include <cmath>
#include <cstdlib>
#include <memory>

#include "fir.cuh"

thread_local std::string g_b2s_last_error;

int32_t b2s_fail(b2s_ctx *ctx, int32_t code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_b2s_last_error = buf;
    if (ctx) ctx->err = buf;
    return code;
}

extern "C" {

int32_t b2s_version(void) { return B2S_VERSION; }

static int32_t ctx_create(int device, void *stream, bool own, b2s_ctx **out) {
    if (!out) return b2s_fail(nullptr, B2S_EINVAL, "b2s_ctx_create: out is NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return b2s_fail(nullptr, B2S_ECUDA, "no CUDA device: %s", cudaGetErrorString(e));
    if (device < 0 || device >= ndev)
        return b2s_fail(nullptr, B2S_EINVAL, "device %d out of range (%d devices)", device, ndev);
    std::unique_ptr<b2s_ctx> guard(new b2s_ctx());      // freed on every early return below
    b2s_ctx *ctx = guard.get();
    ctx->device = device;
    DeviceGuard dg(device);
    cudaDeviceProp prop;
    B2S_CUDA(ctx, cudaGetDeviceProperties(&prop, device));
    ctx->sm_count = prop.multiProcessorCount;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    if (prop.major != 9 || prop.minor != 0) {   // sm_90a code (wgmma) runs on compute capability 9.0 only
        return b2s_fail(nullptr, B2S_EUNSUPPORTED, "device %d is sm_%d%d; libb200sdr is built for sm_90a only",
                        device, prop.major, prop.minor);
    }
    if (!own) {
        ctx->stream = (cudaStream_t)stream;
    } else {
        B2S_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        ctx->owns_stream = true;
    }
    B2S_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking));
    B2S_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking));
    B2S_CUDA(ctx, cudaMalloc((void **)&ctx->d_status, 256));
    B2S_CUDA(ctx, cudaMemsetAsync(ctx->d_status, 0, 256, ctx->stream));
    *out = guard.release();
    return B2S_OK;
}

int32_t b2s_ctx_create(int device, b2s_ctx **out) { return ctx_create(device, nullptr, true, out); }
int32_t b2s_ctx_create_on_stream(int device, void *stream, b2s_ctx **out) {
    return ctx_create(device, stream, false, out);
}

void b2s_ctx_destroy(b2s_ctx *ctx) {
    if (!ctx) return;
    DeviceGuard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->ws_dev) cudaFree(ctx->ws_dev);
    if (ctx->d_status) cudaFree(ctx->d_status);
    if (ctx->s_h2d) cudaStreamDestroy(ctx->s_h2d);
    if (ctx->s_d2h) cudaStreamDestroy(ctx->s_d2h);
    if (ctx->owns_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char *b2s_last_error(const b2s_ctx *ctx) {
    if (ctx && !ctx->err.empty()) return ctx->err.c_str();
    return g_b2s_last_error.c_str();
}

int32_t b2s_ctx_sync(b2s_ctx *ctx) {
    if (!ctx) return b2s_fail(nullptr, B2S_EINVAL, "ctx is NULL");
    DeviceGuard g(ctx->device);
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (ctx->flag_ops) {                       // cross-GPU handshakes were queued: did one of them time out?
        unsigned st = 0;
        B2S_CUDA(ctx, cudaMemcpy(&st, ctx->d_status, sizeof(st), cudaMemcpyDeviceToHost));
        ctx->flag_ops = 0;
        if (st) {
            cudaMemset(ctx->d_status, 0, sizeof(st));
            if (st & 1u)
                return b2s_fail(ctx, B2S_ETIMEOUT, "a cross-GPU flag wait timed out (status 0x%x): the peer never published its chunk", st);
            return b2s_fail(ctx, B2S_ETIMEOUT, "an IIR scan look-back wait timed out (status 0x%x)", st);
        }
    }
    return B2S_OK;
}

void *b2s_ctx_stream(b2s_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }
int32_t b2s_ctx_sm_count(b2s_ctx *ctx) { return ctx ? ctx->sm_count : 0; }
uint64_t b2s_ctx_launch_count(const b2s_ctx *ctx) { return ctx ? ctx->launches.load() : 0; }
uint64_t b2s_ctx_bytes_held(const b2s_ctx *ctx) { return ctx ? ctx->bytes_held.load() : 0; }

int32_t b2s_malloc(b2s_ctx *ctx, size_t bytes, void **dptr) {
    if (!ctx || !dptr) return b2s_fail(ctx, B2S_EINVAL, "b2s_malloc: NULL argument");
    DeviceGuard g(ctx->device);
    cudaError_t e = cudaMalloc(dptr, bytes ? bytes : 1);
    if (e == cudaErrorMemoryAllocation) {
        cudaGetLastError();
        return b2s_fail(ctx, B2S_ENOMEM, "cudaMalloc(%zu) out of memory", bytes);
    }
    B2S_CUDA(ctx, e);
    return B2S_OK;
}
int32_t b2s_free(b2s_ctx *ctx, void *dptr) {
    if (!ctx) return b2s_fail(ctx, B2S_EINVAL, "ctx is NULL");
    DeviceGuard g(ctx->device);
    B2S_CUDA(ctx, cudaFree(dptr));
    return B2S_OK;
}
int32_t b2s_host_alloc(b2s_ctx *ctx, size_t bytes, void **hptr) {
    if (!ctx || !hptr) return b2s_fail(ctx, B2S_EINVAL, "b2s_host_alloc: NULL argument");
    DeviceGuard g(ctx->device);
    B2S_CUDA(ctx, cudaHostAlloc(hptr, bytes ? bytes : 1, cudaHostAllocDefault));
    return B2S_OK;
}
int32_t b2s_host_free(b2s_ctx *ctx, void *hptr) {
    if (!ctx) return b2s_fail(ctx, B2S_EINVAL, "ctx is NULL");
    B2S_CUDA(ctx, cudaFreeHost(hptr));
    return B2S_OK;
}
int32_t b2s_memcpy_h2d(b2s_ctx *ctx, void *dptr, const void *hptr, size_t bytes) {
    if (!ctx) return b2s_fail(ctx, B2S_EINVAL, "ctx is NULL");
    DeviceGuard g(ctx->device);
    B2S_CUDA(ctx, cudaMemcpyAsync(dptr, hptr, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return B2S_OK;
}
int32_t b2s_memcpy_d2h(b2s_ctx *ctx, void *hptr, const void *dptr, size_t bytes) {
    if (!ctx) return b2s_fail(ctx, B2S_EINVAL, "ctx is NULL");
    DeviceGuard g(ctx->device);
    B2S_CUDA(ctx, cudaMemcpyAsync(hptr, dptr, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    return B2S_OK;
}

/* ------------------------------------------------------------------------------------------
 * FIR
 * ---------------------------------------------------------------------------------------- */
// Short filters: the CUDA-core kernel is HBM-bound as well and keeps plain FP32 products, so it stays the
// default below this many taps.  The value is carried over from the previous (B200) tuning; the crossover has not
// been re-measured on H100.
static constexpr size_t kTensorMinTaps = 24;
// Long filters (beyond the tensor kernel's 257 taps) go to the overlap-save FFT kernel.
static constexpr size_t kFftMinTaps = 258;
// Constant tap vectors (boxcar / moving-average / CIC-like filters): every partial-product error of the split-bf16
// tensor path has the same sign there, and on DC-heavy input they add coherently up to ~3e-5 of ||taps||_1 max|x|
// (tests/test_gpu_fir_tensor_structured.py) -- AUTO keeps those on the CUDA cores (exact f32 products).
static bool taps_constant(const b2s_fir *f) {
    if (f->kind == B2S_C32_C32) return false;
    for (size_t i = 1; i < f->ntaps; i++)
        if (f->taps_host[i] != f->taps_host[0]) return false;
    return true;
}
static void resolve_algo(b2s_fir *f) {
    if (f->algo_req == B2S_ALGO_TENSOR && fir_tc_supported(f)) f->algo = B2S_ALGO_TENSOR;
    else if (f->algo_req == B2S_ALGO_FFT && fir_fft_supported(f)) f->algo = B2S_ALGO_FFT;
    else if (f->algo_req == B2S_ALGO_AUTO && fir_tc_supported(f) && f->ntaps >= kTensorMinTaps && !taps_constant(f))
        f->algo = B2S_ALGO_TENSOR;
    else if (f->algo_req == B2S_ALGO_AUTO && fir_fft_supported(f) &&
             (f->ntaps >= kFftMinTaps || (f->kind == B2S_C32_C32 && f->ntaps >= 128)))
        f->algo = B2S_ALGO_FFT;
    else f->algo = B2S_ALGO_DIRECT;
}

static int32_t prepare_algo(b2s_fir *f) {
    if (f->algo == B2S_ALGO_TENSOR) return fir_tc_prepare(f);
    if (f->algo == B2S_ALGO_FFT) return fir_fft_prepare(f);
    return B2S_OK;
}

int32_t b2s_fir_plan(b2s_ctx *ctx, b2s_kind kind, const float *taps, size_t ntaps, size_t decim,
                     b2s_fir **out) {
    if (!ctx || !out || !taps) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_plan: NULL argument");
    *out = nullptr;
    if (ntaps == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_plan: ntaps must be > 0");
    if (decim == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_plan: decim must be > 0");
    if (kind == B2S_F64_F64) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_plan: f64 taps are passed through b2s_fir_plan_f64_f64");
    if (kind != B2S_F32_F32 && kind != B2S_C32_F32 && kind != B2S_C32_C32)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_plan: bad kind %d", (int)kind);
    if (ntaps > (1u << 20) || decim > (1u << 16))
        return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_fir_plan: ntaps/decim too large");
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_fir> f(new b2s_fir());
    f->ctx = ctx; f->kind = kind; f->ntaps = ntaps; f->decim = decim;
    f->taps_host.assign(taps, taps + ntaps * kind_tap_floats(kind));
    B2S_TRY(fir_direct_prepare(f.get()));
    resolve_algo(f.get());
    B2S_TRY(prepare_algo(f.get()));
    *out = f.release();
    return B2S_OK;
}
int32_t b2s_fir_plan_f64_f64(b2s_ctx *ctx, const double *taps, size_t ntaps, size_t decim, b2s_fir **out) {
    if (!ctx || !out || !taps) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_plan_f64_f64: NULL argument");
    *out = nullptr;
    if (ntaps == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_plan: ntaps must be > 0");
    if (decim == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_plan: decim must be > 0");
    if (ntaps > (1u << 20) || decim > (1u << 16)) return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_fir_plan: ntaps/decim too large");
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_fir> f(new b2s_fir());
    f->ctx = ctx; f->kind = B2S_F64_F64; f->ntaps = ntaps; f->decim = decim;
    f->algo_req = f->algo = B2S_ALGO_DIRECT;
    B2S_TRY(fir_f64_prepare(f.get(), taps));
    *out = f.release();
    return B2S_OK;
}
int32_t b2s_fir_plan_f32_f32(b2s_ctx *c, const float *t, size_t n, size_t d, b2s_fir **o) {
    return b2s_fir_plan(c, B2S_F32_F32, t, n, d, o);
}
int32_t b2s_fir_plan_c32_f32(b2s_ctx *c, const float *t, size_t n, size_t d, b2s_fir **o) {
    return b2s_fir_plan(c, B2S_C32_F32, t, n, d, o);
}
int32_t b2s_fir_plan_c32_c32(b2s_ctx *c, const float *t, size_t n, size_t d, b2s_fir **o) {
    return b2s_fir_plan(c, B2S_C32_C32, t, n, d, o);
}

void b2s_fir_destroy(b2s_fir *f) { PlanDeleter<b2s_fir>()(f); }

size_t b2s_fir_length(const b2s_fir *f) { return f ? f->ntaps : 0; }

int32_t b2s_fir_set_algo(b2s_fir *f, b2s_algo algo) {
    if (!f) return b2s_fail(nullptr, B2S_EINVAL, "fir is NULL");
    if (algo < B2S_ALGO_AUTO || algo > B2S_ALGO_FFT)      // B2S_ALGO_SCAN is an IIR algorithm
        return b2s_fail(f->ctx, B2S_EUNSUPPORTED, "FIR filters have the AUTO, DIRECT, TENSOR and FFT algorithms (got %d)", (int)algo);
    if (f->kind == B2S_F64_F64)
        return algo == B2S_ALGO_AUTO || algo == B2S_ALGO_DIRECT ? B2S_OK
               : b2s_fail(f->ctx, B2S_EUNSUPPORTED, "f64 filters only have the CUDA-core form");
    if (algo == B2S_ALGO_TENSOR && !fir_tc_supported(f))
        return b2s_fail(f->ctx, B2S_EUNSUPPORTED,
                        "tensor algorithm needs real taps, 16..257 of them, and a decimation that divides 128 (kind %d, ntaps %zu, decim %zu)",
                        (int)f->kind, f->ntaps, f->decim);
    if (algo == B2S_ALGO_FFT && !fir_fft_supported(f))
        return b2s_fail(f->ctx, B2S_EUNSUPPORTED,
                        "FFT algorithm needs Complex<f32> samples, 64..2049 taps and decim == 1 (kind %d, ntaps %zu, decim %zu)",
                        (int)f->kind, f->ntaps, f->decim);
    f->algo_req = algo;
    resolve_algo(f);
    DeviceGuard g(f->ctx->device);
    return prepare_algo(f);
}
int32_t b2s_fir_get_algo(const b2s_fir *f) { return f ? (int32_t)f->algo : B2S_EINVAL; }

// (consumed, produced, status) of DecimatingFirFilter (decimating_fir.rs:70-78,:94); with
// decim == 1 this is exactly FirFilter's triple (fir.rs:69-74,:90).
static void fir_counts(const b2s_fir *f, size_t n_in, size_t n_out_cap, size_t *consumed,
                       size_t *produced, int32_t *status) {
    const size_t filterable = sat_sub(n_in + 1, f->ntaps);
    const size_t consumable = filterable / f->decim;
    size_t n;
    int32_t st;
    if (consumable > n_out_cap) { n = n_out_cap; st = B2S_INSUFFICIENT_OUTPUT; }
    else if (consumable == n_out_cap) { n = n_out_cap; st = B2S_BOTH_SUFFICIENT; }
    else { n = consumable; st = B2S_INSUFFICIENT_INPUT; }
    *consumed = n * f->decim; *produced = n; *status = st;
}

static int32_t fir_launch(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out,
                          cudaStream_t stream) {
    if (f->kind == B2S_F64_F64) return fir_f64_launch(f, d_in, n_in, d_out, n_out, stream);
    // SMALL slices under AUTO: the tensor kernel has a fixed per-launch cost (Toeplitz fill, one persistent CTA per
    // SM) that the CUDA-core kernel does not pay; the latter's time grows with n_out * ntaps (per_tap: estimated
    // seconds per sample-tap, scripts/small_sweep.py; carried over from the previous (B200) tuning, not re-measured
    // on H100).  Below ~10 us of estimated CUDA-core time the direct form is used.  An explicit B2S_ALGO_TENSOR request is always honoured.
    if (f->algo == B2S_ALGO_TENSOR && f->algo_req == B2S_ALGO_AUTO) {
        const double per_tap = f->kind == B2S_F32_F32 ? 6.9e-14 : 1.15e-13;
        if ((double)n_out * (double)f->ntaps * per_tap < 10e-6) return fir_direct_launch(f, d_in, n_in, d_out, n_out, stream);
    }
    if (f->algo == B2S_ALGO_TENSOR) return fir_tc_launch(f, d_in, n_in, d_out, n_out, stream);
    if (f->algo == B2S_ALGO_FFT) return fir_fft_launch(f, d_in, n_in, d_out, n_out, stream);
    return fir_direct_launch(f, d_in, n_in, d_out, n_out, stream);
}

int32_t b2s_fir_exec(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                     size_t *consumed, size_t *produced, int32_t *status) {
    if (!f || !consumed || !produced || !status)
        return b2s_fail(f ? f->ctx : nullptr, B2S_EINVAL, "b2s_fir_exec: NULL argument");
    fir_counts(f, n_in, n_out_cap, consumed, produced, status);
    if (*produced == 0) return B2S_OK;
    if (!d_in || !d_out) return b2s_fail(f->ctx, B2S_EINVAL, "b2s_fir_exec: NULL buffer");
    DeviceGuard g(f->ctx->device);
    NvtxRange nvtx("b2s_fir_exec");
    return fir_launch(f, d_in, n_in, d_out, *produced, f->ctx->stream);
}

// Host-slice drop-in for Filter::filter.  The input is cut into chunks of CH outputs; chunk c
// needs input items [c*CH*D, c*CH*D + CH*D + ntaps - 1) (overlap re-read from the host slice,
// the same history the reference's ring keeps in place, blocks/fir.rs:49).  Three-stage
// pipeline over two device slots: H2D on s_h2d, kernel on the context stream, D2H on s_d2h.
int32_t b2s_fir_filter_host(b2s_fir *f, const void *h_in, size_t n_in, void *h_out, size_t n_out_cap,
                            size_t *consumed, size_t *produced, int32_t *status) {
    if (!f || !consumed || !produced || !status)
        return b2s_fail(f ? f->ctx : nullptr, B2S_EINVAL, "b2s_fir_filter_host: NULL argument");
    b2s_ctx *ctx = f->ctx;
    fir_counts(f, n_in, n_out_cap, consumed, produced, status);
    const size_t n_out = *produced;
    if (n_out == 0) return B2S_OK;
    if (!h_in || !h_out) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_filter_host: NULL buffer");
    DeviceGuard g(ctx->device);
    // One host pipeline per context at a time: the workspace, the side streams and the events are shared by every
    // plan of the context (Filter::filter is re-entrant in the reference; here concurrent callers queue up).
    std::lock_guard<std::mutex> lk(ctx->host_mu);

    const size_t isz = kind_in_bytes(f->kind), D = f->decim, N = f->ntaps;
    constexpr int NSLOT = 4;
    // chunk: ~32 MiB of input per slot (B2S_HOST_CHUNK_MB overrides), whole multiples of the direct kernel's
    // 1024-output tile.  Shorter chunks shorten the un-overlapped first H2D / last D2H but lose more to
    // per-copy overhead.
    static const size_t chunk_mb = [] { const char *e = getenv("B2S_HOST_CHUNK_MB"); const long v = e ? atol(e) : 32; return (size_t)(v > 0 ? v : 32); }();
    size_t CH = round_up(std::max<size_t>((chunk_mb << 20) / (isz * D), 1024), 1024);
    if (CH > n_out) CH = round_up(n_out, 1024);
    const size_t in_items = CH * D + N - 1;
    const size_t in_bytes = round_up(in_items * isz, 256), out_bytes = round_up(CH * isz, 256);
    const size_t need = NSLOT * (in_bytes + out_bytes);
    if (ctx->ws_bytes < need) {
        if (ctx->ws_dev) {
            // nothing queued on any of the three streams may still touch the old workspace
            B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            B2S_CUDA(ctx, cudaStreamSynchronize(ctx->s_h2d));
            B2S_CUDA(ctx, cudaStreamSynchronize(ctx->s_d2h));
            cudaFree(ctx->ws_dev);
        }
        ctx->ws_dev = nullptr; ctx->ws_bytes = 0;
        cudaError_t e = cudaMalloc(&ctx->ws_dev, need);
        if (e != cudaSuccess) { cudaGetLastError(); return b2s_fail(ctx, B2S_ENOMEM, "workspace %zu B", need); }
        ctx->ws_bytes = need;
    }
    char *base = (char *)ctx->ws_dev;
    if (!ctx->hev_ready) {
        for (int i = 0; i < 3 * NSLOT + 1; i++) B2S_CUDA(ctx, cudaEventCreateWithFlags(&ctx->hev[i], cudaEventDisableTiming));
        ctx->hev_ready = true;
    }
    cudaEvent_t *ev_in = ctx->hev, *ev_k = ctx->hev + NSLOT, *ev_out = ctx->hev + 2 * NSLOT, ev0 = ctx->hev[3 * NSLOT];
    int32_t rc = B2S_OK;
    const size_t nchunks = ceil_div(n_out, CH);
    // the copies must not start before work already queued on the context stream that may
    // still use the workspace
    B2S_CUDA(ctx, cudaEventRecord(ev0, ctx->stream));
    B2S_CUDA(ctx, cudaStreamWaitEvent(ctx->s_h2d, ev0, 0));
    B2S_CUDA(ctx, cudaStreamWaitEvent(ctx->s_d2h, ev0, 0));
    nvtx_push("b2s_fir_filter_host");
    for (size_t c = 0; c < nchunks && rc == B2S_OK; c++) {
        const int s = (int)(c % NSLOT);
        char *din = base + (size_t)s * (in_bytes + out_bytes), *dout = din + in_bytes;
        const size_t k0 = c * CH, nk = std::min(CH, n_out - k0);
        const size_t i0 = k0 * D, ni = nk * D + N - 1;     // <= n_in by construction
        if (c >= NSLOT) {
            // slot reuse: the H2D may overwrite din only after kernel c-NSLOT ran, and the
            // kernel may overwrite dout only after D2H c-NSLOT finished
            cudaStreamWaitEvent(ctx->s_h2d, ev_k[s], 0);
            cudaStreamWaitEvent(ctx->stream, ev_out[s], 0);
        }
        cudaMemcpyAsync(din, (const char *)h_in + i0 * isz, ni * isz, cudaMemcpyHostToDevice, ctx->s_h2d);
        cudaEventRecord(ev_in[s], ctx->s_h2d);
        cudaStreamWaitEvent(ctx->stream, ev_in[s], 0);
        rc = fir_launch(f, din, ni, dout, nk, ctx->stream);
        cudaEventRecord(ev_k[s], ctx->stream);
        cudaStreamWaitEvent(ctx->s_d2h, ev_k[s], 0);
        cudaMemcpyAsync((char *)h_out + k0 * isz, dout, nk * isz, cudaMemcpyDeviceToHost, ctx->s_d2h);
        cudaEventRecord(ev_out[s], ctx->s_d2h);
    }
    cudaError_t e1 = cudaStreamSynchronize(ctx->s_d2h);
    cudaError_t e2 = cudaStreamSynchronize(ctx->stream);
    cudaError_t e3 = cudaStreamSynchronize(ctx->s_h2d);
    nvtx_pop();
    if (rc != B2S_OK) return rc;
    B2S_CUDA(ctx, e1); B2S_CUDA(ctx, e2); B2S_CUDA(ctx, e3);
    B2S_CUDA(ctx, cudaGetLastError());
    return B2S_OK;
}

// ≙ Filter::filter on the logical slice  hist[0..n_hist) ++ in[0..n_in)  (include/b200sdr.h).
int32_t b2s_fir_exec_hist(b2s_fir *f, const void *d_hist, size_t n_hist, const void *d_in, size_t n_in,
                          void *d_out, size_t n_out_cap, const b2s_handshake *hs, size_t *consumed, size_t *produced,
                          int32_t *status) {
    if (!f || !consumed || !produced || !status)
        return b2s_fail(f ? f->ctx : nullptr, B2S_EINVAL, "b2s_fir_exec_hist: NULL argument");
    b2s_ctx *ctx = f->ctx;
    if (n_hist && !d_hist) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_exec_hist: NULL history");
    fir_counts(f, n_hist + n_in, n_out_cap, consumed, produced, status);
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_fir_exec_hist");
    cudaStream_t st = ctx->stream;
    FirHist h;
    h.d_hist = d_hist; h.n_hist = n_hist;
    if (hs) {
        h.publish_flag = hs->publish_flag; h.publish_value = hs->publish_value;
        h.wait_flag = hs->wait_flag; h.wait_value = hs->wait_value;
        h.done_flag = hs->done_flag; h.done_value = hs->done_value;
    }
    // the flag protocol with separate (one-thread) kernels, for everything but the fused tensor launch
    auto publish = [&]() -> int32_t { return h.publish_flag ? peer_flag_set_launch(ctx, h.publish_flag, h.publish_value, st) : B2S_OK; };
    auto wait = [&]() -> int32_t { return h.wait_flag ? peer_flag_wait_launch(ctx, h.wait_flag, h.wait_value, st) : B2S_OK; };
    auto done = [&]() -> int32_t { return h.done_flag ? peer_flag_set_launch(ctx, h.done_flag, h.done_value, st) : B2S_OK; };
    int32_t rc;
    if (*produced == 0) {                          // nothing to compute: still honour the protocol
        if ((rc = publish()) || (rc = wait()) || (rc = done())) return rc;
        return B2S_OK;
    }
    if (!d_in || !d_out) return b2s_fail(ctx, B2S_EINVAL, "b2s_fir_exec_hist: NULL buffer");
    if (f->algo == B2S_ALGO_TENSOR && f->kind != B2S_F64_F64 && (n_hist || h.publish_flag)) {
        rc = fir_tc_launch_hist(f, &h, d_in, n_in, d_out, *produced, st);   // fused: publish, wait, fetch, done in the kernel
        if (rc != B2S_EAGAIN) return rc;
    }
    // every other path wants one contiguous slice: install the history in the n_hist items in front of d_in (the
    // caller guarantees they are writable scratch of the same allocation -- a ring slot's halo region)
    if ((rc = publish()) || (rc = wait())) return rc;
    const size_t isz = kind_in_bytes(f->kind);
    char *dst = (char *)const_cast<void *>(d_in) - n_hist * isz;
    if (n_hist && dst != (const char *)d_hist)
        B2S_CUDA(ctx, cudaMemcpyAsync(dst, d_hist, n_hist * isz, cudaMemcpyDefault, st));
    if ((rc = done())) return rc;
    return fir_launch(f, dst, n_hist + n_in, d_out, *produced, st);
}

}  // extern "C"
