// common.cuh -- context object, error plumbing and small device helpers shared by all
// translation units of libb200sdr.so.
#pragma once

#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "b200sdr.h"

struct b2s_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool owns_stream = false;
    // side streams + events for the host-slice pipeline (b2s_fir_filter_host)
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    int sm_count = 0;
    size_t smem_optin = 0;
    std::atomic<uint64_t> launches{0};
    std::string err;
    // workspace for *_host calls (grown on demand, freed with the context)
    void *ws_dev = nullptr;
    size_t ws_bytes = 0;
    cudaEvent_t hev[16] = {};      // events of the host-slice pipeline, created once
    bool hev_ready = false;
    std::mutex host_mu;            // serialises the *_host pipelines that share the workspace and side streams
    // device status word (bit0: a cross-GPU flag wait timed out); checked by b2s_ctx_sync when flag_ops > 0
    unsigned *d_status = nullptr;
    uint64_t flag_ops = 0;
    // device + pinned bytes held by the Bufs of the objects created on this context (b2s_ctx_bytes_held)
    std::atomic<uint64_t> bytes_held{0};
};

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per DEVICE and a process may hold contexts on several: the
// PerDeviceOnce of each kernel in smem_optin (below) remembers which devices have been opted in.
struct PerDeviceOnce {
    std::atomic<uint64_t> mask{0};
    bool need(int dev) const { return ((mask.load(std::memory_order_acquire) >> (dev & 63)) & 1ull) == 0; }
    void done(int dev) { mask.fetch_or(1ull << (dev & 63), std::memory_order_release); }
};

#ifdef __CUDACC__
__device__ __forceinline__ void mac(float &acc, float x, float t) { acc = fmaf(x, t, acc); }
// acc += x * t for a Complex<f32> sample and a REAL tap: two IEEE fused multiply-adds (sm_90 has no packed FFMA2).
__device__ __forceinline__ void mac(float2 &acc, float2 x, float t) {
    acc.x = fmaf(x.x, t, acc.x);
    acc.y = fmaf(x.y, t, acc.y);
}
// Complex tap: re = xr*tr - xi*ti, im = xr*ti + xi*tr (fir.rs:257-276)
__device__ __forceinline__ void mac(float2 &acc, float2 x, float2 t) {
    acc.x = fmaf(x.x, t.x, acc.x);
    acc.x = fmaf(-x.y, t.y, acc.x);
    acc.y = fmaf(x.x, t.y, acc.y);
    acc.y = fmaf(x.y, t.x, acc.y);
}

template <typename S> __device__ __forceinline__ S zero_of();
template <> __device__ __forceinline__ float zero_of<float>() { return 0.0f; }
template <> __device__ __forceinline__ float2 zero_of<float2>() { return make_float2(0.f, 0.f); }

// cp.async (LDGSTS): global -> shared copies that hold no registers while in flight.  .ca also caches the line in L1,
// .cg only in L2.  The forms with `valid` zero-fill the destination when it is false (src-size 0); src must then still
// be a mapped address.  commit() closes a group of the thread's copies; wait<N>() returns when at most N groups are
// still in flight (the thread's own copies only: a barrier publishes them to the CTA).
namespace cp_async {
__device__ __forceinline__ void ca4(float *dst_smem, const float *src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst_smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(src) : "memory");
}
__device__ __forceinline__ void ca4(float *dst_smem, const float *src, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst_smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(valid ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cg16(void *dst_smem, const void *src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst_smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src) : "memory");
}
__device__ __forceinline__ void cg16(void *dst_smem, const void *src, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst_smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
}  // namespace cp_async
#endif

extern thread_local std::string g_b2s_last_error;

int32_t b2s_fail(b2s_ctx *ctx, int32_t code, const char *fmt, ...);

#define B2S_CUDA(ctx, expr)                                                                   \
    do {                                                                                      \
        cudaError_t e__ = (expr);                                                             \
        if (e__ != cudaSuccess)                                                               \
            return b2s_fail((ctx), B2S_ECUDA, "%s failed: %s (%s:%d)", #expr,                 \
                            cudaGetErrorString(e__), __FILE__, __LINE__);                     \
    } while (0)

#define B2S_CHECK_LAUNCH(ctx)                                                                 \
    do {                                                                                      \
        (ctx)->launches.fetch_add(1, std::memory_order_relaxed);                              \
        B2S_CUDA((ctx), cudaGetLastError());                                                  \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

#define B2S_TRY(expr)                                                                         \
    do {                                                                                      \
        const int32_t rc__ = (expr);                                                          \
        if (rc__ != B2S_OK) return rc__;                                                      \
    } while (0)

// Opt kernel K in to `bytes` of dynamic shared memory on the context's device, once per device; with `resident`, also
// report how many CTAs of K at `threads` threads and `bytes` fit one SM (queried once per device, at least 1).  Every
// call site of one K passes the same figures.
template <auto K>
int32_t smem_optin(b2s_ctx *ctx, size_t bytes, int threads = 0, int *resident = nullptr) {
    static PerDeviceOnce optin;
    static std::atomic<int> ctas[64];
    if (bytes > 48 * 1024 && optin.need(ctx->device)) {
        B2S_CUDA(ctx, cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        optin.done(ctx->device);
    }
    if (resident) {
        std::atomic<int> &n = ctas[ctx->device & 63];
        int r = n.load(std::memory_order_relaxed);
        if (!r) {
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&r, K, threads, bytes) != cudaSuccess || r < 1) { cudaGetLastError(); r = 1; }
            n.store(r, std::memory_order_relaxed);
        }
        *resident = r;
    }
    return B2S_OK;
}

// Ownership: every buffer and sub-plan an object allocates is freed by its owner's destructor.  A Buf owns device
// (or pinned host) memory and counts it in its context's bytes_held; a plan under construction lives in a PlanPtr
// until it is handed out through *out, so an early return frees whatever was built so far.
enum class Mem { Device, Pinned };

template <typename T, Mem M = Mem::Device>
class Buf {
  public:
    Buf() = default;
    Buf(Buf &&o) noexcept { swap(o); }
    Buf &operator=(Buf &&o) noexcept {
        Buf(std::move(o)).swap(*this);
        return *this;
    }
    ~Buf() { reset(); }

    T *get() const { return p_; }
    size_t size() const { return n_; }   // elements
    explicit operator bool() const { return p_ != nullptr; }

    void reset() {
        if (!ctx_) return;
        if (M == Mem::Device) cudaFree(p_);
        else cudaFreeHost(p_);
        ctx_->bytes_held -= n_ * sizeof(T);
        ctx_ = nullptr; p_ = nullptr; n_ = 0;
    }
    // n uninitialised elements in place of what the buffer held
    int32_t alloc(b2s_ctx *ctx, size_t n, const char *what) {
        reset();
        void *p = nullptr;
        const cudaError_t e = M == Mem::Device ? cudaMalloc(&p, n * sizeof(T))
                                               : cudaHostAlloc(&p, n * sizeof(T), cudaHostAllocDefault);
        if (e != cudaSuccess) {
            cudaGetLastError();   // reported here, not again by the next launch check
            return b2s_fail(ctx, B2S_ENOMEM, "%s: %zu bytes: %s", what, n * sizeof(T), cudaGetErrorString(e));
        }
        ctx_ = ctx; p_ = static_cast<T *>(p); n_ = n;
        ctx->bytes_held += n * sizeof(T);
        return B2S_OK;
    }
    // alloc, then copy n elements from `host` on the context stream (the caller synchronises before `host` dies)
    int32_t upload(b2s_ctx *ctx, const T *host, size_t n, const char *what) {
        B2S_TRY(alloc(ctx, n, what));
        B2S_CUDA(ctx, cudaMemcpyAsync(p_, host, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
        return B2S_OK;
    }
    // grow-on-demand workspace: nothing to do while it holds n elements; otherwise wait until the context stream no
    // longer uses the old memory and allocate n (the buffer is left empty if that fails)
    int32_t reserve(b2s_ctx *ctx, size_t n, const char *what) {
        if (n_ >= n) return B2S_OK;
        B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return alloc(ctx, n, what);
    }

  private:
    void swap(Buf &o) noexcept {
        std::swap(ctx_, o.ctx_); std::swap(p_, o.p_); std::swap(n_, o.n_);
    }
    b2s_ctx *ctx_ = nullptr;
    T *p_ = nullptr;
    size_t n_ = 0;
};

// Every b2s_*_destroy: wait for the plan's context stream (queued work may still use the plan's memory), then
// delete the plan on its device.
template <typename P> struct PlanDeleter {
    void operator()(P *p) const {
        if (!p) return;
        DeviceGuard g(p->ctx->device);
        cudaStreamSynchronize(p->ctx->stream);
        delete p;
    }
};
template <typename P> using PlanPtr = std::unique_ptr<P, PlanDeleter<P>>;

// peer.cu: NVTX ranges (visible to nsys / ncu --nvtx) and the cross-GPU flag kernels
void nvtx_push(const char *name);
void nvtx_pop();
struct NvtxRange { explicit NvtxRange(const char *n) { nvtx_push(n); } ~NvtxRange() { nvtx_pop(); } };
int32_t peer_flag_set_launch(b2s_ctx *ctx, unsigned *flag, unsigned value, cudaStream_t st);
int32_t peer_flag_wait_launch(b2s_ctx *ctx, const unsigned *flag, unsigned value, cudaStream_t st);

static inline size_t sat_sub(size_t a, size_t b) { return a > b ? a - b : 0; }
static inline size_t ceil_div(size_t a, size_t b) { return (a + b - 1) / b; }
static inline size_t round_up(size_t a, size_t b) { return ceil_div(a, b) * b; }

// slice checks of the exec calls: byte ranges [p, p + pb) and [q, q + qb) share a byte (empty ranges share none)
static inline bool overlap(const void *p, size_t pb, const void *q, size_t qb) {
    const uintptr_t a = (uintptr_t)p, b = (uintptr_t)q;
    return pb && qb && a < b + qb && b < a + pb;
}
// an output may be disjoint from an input, or lie exactly on it with the same item size (in place)
static inline bool bad_alias(const void *out, size_t ob, size_t oi, const void *in, size_t ib, size_t ii) {
    if (!overlap(out, ob, in, ib)) return false;
    return !(out == in && oi == ii);
}
static inline bool word_aligned(const void *p) { return ((uintptr_t)p & 3) == 0; }

static inline size_t kind_in_bytes(b2s_kind k) { return k == B2S_F32_F32 ? 4 : 8; }   // F64_F64: 8 as well
static inline size_t kind_tap_floats(b2s_kind k) { return k == B2S_C32_C32 ? 2 : 1; }
