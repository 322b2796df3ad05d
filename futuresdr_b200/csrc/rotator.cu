// rotator.cu -- futuredsp::Rotator (crates/futuredsp/src/rotator.rs:13-48), the band-pass tap
// construction of XlatingFir (src/blocks/xlating_fir.rs:72-103) -- SURVEY.md §8f row 1 -- and the SSB example's
// oscillator closures (examples/ssb/{transmit,receive}.rs), which run the same recurrence (b2s_mixer, DESIGN §4.18).
//
// The reference rotator is an f32 product recurrence with NO renormalisation:
//     phase *= phase_incr;  out = in * phase          (per sample, num_complex Mul)
// |phase_incr| differs from 1 by up to an ulp, so |phase| drifts like (1+d)^n: evaluating
// incr^n in closed form would leave the 1e-5 band after ~10^2..10^5 samples.  To stay identical
// to the reference the recurrence itself is replayed: it does not depend on the data, so the host
// runs it once per call (plain f32 ops, no contraction) and records the phase every 8 samples
// (1 byte/sample of extra traffic); on the device each thread re-derives its sample's phase from
// the record with the same IEEE operations (__fmul_rn/__fsub_rn/__fadd_rn) -- bit-identical
// phases, data-parallel rotation.  The replay runs AHEAD of the stream on a worker thread (below), so a call only
// waits for it when the stream is sustained above the replay rate (~0.4 Gsamples/s of rotator input).
#include <cmath>
#include <condition_variable>
#include <thread>

#include "chunks.cuh"

namespace {
constexpr int kRotSub = 8;                      // samples per recorded phase
constexpr size_t kRingRecs = 4u << 20;          // run-ahead window: 4 Mi records = 32 Mi samples (32 MiB pinned)
constexpr size_t kBatchRecs = 1u << 14;         // the worker publishes its progress every 16 Ki records
}

// The recurrence is data-independent, so a WORKER THREAD runs it ahead of the stream: it fills a pinned ring with the
// phase before every 8th sample of the (infinite) stream and an exec call only waits if the stream has outrun it
// (sustained ~0.4 Gsamples/s, the speed of the dependent f32 multiply-add chain on one core -- the same chain the
// reference's own rotate() runs); the records of a call travel with one or two async H2D copies.
struct b2s_rotator {
    b2s_ctx *ctx = nullptr;
    float incr[2] = {1.f, 0.f};
    Buf<float2, Mem::Pinned> h_ring;             // kRingRecs records; record r lives at r % kRingRecs
    Buf<float2> d_recs;                          // records of the calls in flight on the device (two halves)
    int half = 0;
    cudaEvent_t ev[2] = {nullptr, nullptr};      // H2D of half i done -> its ring span may be overwritten
    uint64_t span_end[2] = {0, 0};               // one past the last record each half's copy read
    uint64_t pos = 0;                            // samples rotated so far (stream position)
    // worker
    std::thread worker;
    std::mutex mu;
    std::condition_variable cv;
    uint64_t produced = 0;                       // records computed (absolute)
    uint64_t released = 0;                       // records below this may be overwritten
    uint64_t epoch = 0;                          // bumped by reset
    bool quit = false;

    void stop_worker() {
        { std::lock_guard<std::mutex> lk(mu); quit = true; }
        cv.notify_all();
        if (worker.joinable()) worker.join();
    }
    ~b2s_rotator() {
        stop_worker();
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    }
};

// The SSB example's oscillator closures (b2s_mix_op): the same replay, a different epilogue per sample.
struct b2s_mixer {
    b2s_ctx *ctx = nullptr;
    b2s_mix_op op = B2S_MIX_ROTATE_C32;
    float param = 1.f;
    b2s_rotator rot;
};

namespace {

void rotator_worker(b2s_rotator *r) {
    uint64_t epoch = ~0ull, next = 0;
    float pr = 1.f, pi = 0.f;
    const float ir = r->incr[0], ii = r->incr[1];
    for (;;) {
        uint64_t limit;
        {
            std::unique_lock<std::mutex> lk(r->mu);
            r->cv.wait(lk, [&] { return r->quit || r->epoch != epoch || r->produced < r->released + kRingRecs; });
            if (r->quit) return;
            if (r->epoch != epoch) { epoch = r->epoch; next = 0; pr = 1.f; pi = 0.f; r->produced = 0; }   // Rotator::new
            limit = std::min<uint64_t>(r->released + kRingRecs, next + kBatchRecs);
        }
        // host replay of the recurrence: plain binary32 SSE operations (host code is built with -ffp-contract=off and
        // without -ffast-math, so every product and sum is rounded separately) -- rotator.rs:26, num_complex Mul
        for (; next < limit; next++) {
            r->h_ring.get()[next % kRingRecs] = make_float2(pr, pi);
            for (int k = 0; k < kRotSub; k++) {
                const float a = pr * ir, b = pi * ii, c = pr * ii, d = pi * ir;
                pr = a - b; pi = c + d;
            }
        }
        {
            std::lock_guard<std::mutex> lk(r->mu);
            if (r->epoch == epoch) r->produced = next;
        }
        r->cv.notify_all();
    }
}

__device__ __forceinline__ float2 cmul_rn(float2 a, float2 b) {       // num_complex Mul, un-fused
    return make_float2(__fsub_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)),
                       __fadd_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}

// What a sample becomes once its phase is known: the closures `osc *= shift; f(v, osc)` differ only in f.
struct EpiRotate {                                                     // v * osc (rotator.rs:45, transmit.rs:104-107)
    using Out = float2;
    __device__ __forceinline__ float2 operator()(float2 v, float2 p) const { return cmul_rn(v, p); }
};
struct EpiRotateScale {                                                // v * osc * s, Complex * f32 per part (receive.rs:63-66)
    using Out = float2;
    float s;
    __device__ __forceinline__ float2 operator()(float2 v, float2 p) const {
        const float2 t = cmul_rn(v, p);
        return make_float2(__fmul_rn(t.x, s), __fmul_rn(t.y, s));
    }
};
struct EpiWeaver {                                                     // s * (v.re*osc.re + v.im*osc.im) (receive.rs:78-83)
    using Out = float;
    float s;
    __device__ __forceinline__ float operator()(float2 v, float2 p) const {
        return __fmul_rn(s, __fadd_rn(__fmul_rn(v.x, p.x), __fmul_rn(v.y, p.y)));
    }
};

// sample s of the call is sample (off + s) of the record span: record (off + s) / 8, then (off + s) % 8 + 1 steps
template <class Epi>
__global__ void rotator_kernel(const float2 *__restrict__ in, typename Epi::Out *__restrict__ out,
                               const float2 *__restrict__ recs, float2 incr, long long n, int off, Epi epi) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += stride) {
        const long long a = s + off;
        float2 p = recs[a / kRotSub];
        const int j = (int)(a % kRotSub);
#pragma unroll
        for (int i = 0; i < kRotSub; i++)
            if (i <= j) p = cmul_rn(p, incr);                          // phase *= phase_incr, (j+1) times
        out[s] = epi(in[s], p);
    }
}

int32_t replay_init(b2s_rotator *r, b2s_ctx *ctx, float phase_incr) {
    r->ctx = ctx;
    // Complex32::from_polar(1.0, phase_incr) = (1.0 * cos, 1.0 * sin) in f32 (rotator.rs:17)
    r->incr[0] = 1.0f * std::cos(phase_incr);
    r->incr[1] = 1.0f * std::sin(phase_incr);
    B2S_TRY(r->h_ring.alloc(ctx, kRingRecs, "rotator: pinned record ring"));
    for (int i = 0; i < 2; i++) B2S_CUDA(ctx, cudaEventCreateWithFlags(&r->ev[i], cudaEventDisableTiming));
    r->worker = std::thread(rotator_worker, r);
    return B2S_OK;
}

int32_t replay_reset(b2s_rotator *r) {
    DeviceGuard g(r->ctx->device);
    // copies of the old sequence may still be reading the ring
    B2S_CUDA(r->ctx, cudaStreamSynchronize(r->ctx->stream));
    { std::lock_guard<std::mutex> lk(r->mu); r->epoch++; r->produced = 0; r->released = 0; }
    r->cv.notify_all();
    r->pos = 0; r->span_end[0] = r->span_end[1] = 0;
    return B2S_OK;
}

// n > 0 samples of the stream through `epi`, each with the phase the recurrence gives it
template <class Epi>
int32_t replay_exec(b2s_rotator *r, const float2 *in, typename Epi::Out *out, size_t n, Epi epi) {
    b2s_ctx *ctx = r->ctx;
    DeviceGuard g(ctx->device);
    // pieces of at most a quarter of the ring, so that the worker can keep running ahead while a piece is in flight
    const size_t piece_max = (kRingRecs / 4) * kRotSub;
    const size_t d_need = std::min(n, piece_max) / kRotSub + 2;
    B2S_TRY(r->d_recs.reserve(ctx, 2 * d_need, "rotator records"));
    const size_t d_cap = r->d_recs.size() / 2;
    size_t done = 0;
    while (done < n) {
        const size_t m = std::min(n - done, piece_max);
        const uint64_t a0 = r->pos, a1 = r->pos + m;               // absolute samples [a0, a1)
        const uint64_t rec0 = a0 / kRotSub, rec1 = (a1 - 1) / kRotSub + 1;
        const int h = r->half;
        // (the device half we are about to overwrite was last read by the kernel two pieces ago: stream order covers it)
        // Ring space: once the H2D of an earlier piece has completed, the records below that piece's start are free.
        // Poll first; block on the event only if the worker is actually starved for space.
        auto harvest = [&](int hh, bool block) -> int32_t {
            if (!r->span_end[hh]) return B2S_OK;
            cudaError_t e = block ? cudaEventSynchronize(r->ev[hh]) : cudaEventQuery(r->ev[hh]);
            if (e == cudaErrorNotReady) { cudaGetLastError(); return B2S_OK; }
            B2S_CUDA(ctx, e);
            { std::lock_guard<std::mutex> lk(r->mu); r->released = std::max(r->released, r->span_end[hh]); }
            r->span_end[hh] = 0;
            r->cv.notify_all();
            return B2S_OK;
        };
        for (int hh = 0; hh < 2; hh++) { const int32_t rc = harvest(hh, false); if (rc) return rc; }
        for (;;) {
            std::unique_lock<std::mutex> lk(r->mu);                  // only blocks when the stream outran the worker
            if (r->produced >= rec1) break;
            if (r->released + kRingRecs >= rec1) { r->cv.wait(lk, [&] { return r->produced >= rec1; }); break; }
            lk.unlock();                                             // the worker is out of ring space: wait for a copy
            for (int hh = 0; hh < 2; hh++) { const int32_t rc = harvest(hh, true); if (rc) return rc; }
            std::lock_guard<std::mutex> lk2(r->mu);
            if (r->released + kRingRecs < rec1) return b2s_fail(ctx, B2S_ESTATE, "rotator: record ring accounting");
        }
        float2 *drec = r->d_recs.get() + (size_t)h * d_cap;
        const size_t i0 = rec0 % kRingRecs, cnt = rec1 - rec0;
        const size_t first = std::min(cnt, kRingRecs - i0);
        B2S_CUDA(ctx, cudaMemcpyAsync(drec, r->h_ring.get() + i0, first * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
        if (cnt > first)
            B2S_CUDA(ctx, cudaMemcpyAsync(drec + first, r->h_ring.get(), (cnt - first) * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
        B2S_CUDA(ctx, cudaEventRecord(r->ev[h], ctx->stream));
        r->span_end[h] = rec0;                                      // records below rec0 are never needed again
        rotator_kernel<Epi><<<grid_for(ctx, m, 16), kThreads, 0, ctx->stream>>>(
            in + done, out + done, drec, make_float2(r->incr[0], r->incr[1]), (long long)m, (int)(a0 % kRotSub), epi);
        B2S_CHECK_LAUNCH(ctx);
        r->pos = a1; r->half ^= 1; done += m;
    }
    return B2S_OK;
}

}  // namespace

extern "C" {

int32_t b2s_rotator_create(b2s_ctx *ctx, float phase_incr, b2s_rotator **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_rotator_create: NULL argument");
    *out = nullptr;
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_rotator> r(new b2s_rotator());
    B2S_TRY(replay_init(r.get(), ctx, phase_incr));
    *out = r.release();
    return B2S_OK;
}

void b2s_rotator_destroy(b2s_rotator *r) {
    if (r) r->stop_worker();
    PlanDeleter<b2s_rotator>()(r);
}

int32_t b2s_rotator_reset(b2s_rotator *r) {
    if (!r) return b2s_fail(nullptr, B2S_EINVAL, "rotator is NULL");
    return replay_reset(r);
}

// ≙ Rotator::rotate (rotator.rs:32-47); d_in == d_out is rotate_inplace (:24-29)
int32_t b2s_rotator_exec(b2s_rotator *r, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                         size_t *processed, int32_t *status) {
    if (!r || !processed || !status) return b2s_fail(r ? r->ctx : nullptr, B2S_EINVAL, "b2s_rotator_exec: NULL argument");
    size_t n;
    if (n_in > n_out_cap) { n = n_out_cap; *status = B2S_INSUFFICIENT_OUTPUT; }
    else if (n_in == n_out_cap) { n = n_out_cap; *status = B2S_BOTH_SUFFICIENT; }
    else { n = n_in; *status = B2S_INSUFFICIENT_INPUT; }
    *processed = n;
    if (n == 0) return B2S_OK;
    if (!d_in || !d_out) return b2s_fail(r->ctx, B2S_EINVAL, "b2s_rotator_exec: NULL buffer");
    NvtxRange nvtx("b2s_rotator_exec");
    return replay_exec(r, (const float2 *)d_in, (float2 *)d_out, n, EpiRotate{});
}

int32_t b2s_mixer_create(b2s_ctx *ctx, b2s_mix_op op, float phase_incr, float param, b2s_mixer **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_mixer_create: NULL argument");
    *out = nullptr;
    if ((int)op < 0 || (int)op > (int)B2S_MIX_WEAVER_F32) return b2s_fail(ctx, B2S_EINVAL, "b2s_mixer_create: bad op %d", (int)op);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_mixer> m(new b2s_mixer());
    m->ctx = ctx; m->op = op; m->param = param;
    B2S_TRY(replay_init(&m->rot, ctx, phase_incr));
    *out = m.release();
    return B2S_OK;
}

void b2s_mixer_destroy(b2s_mixer *m) {
    if (m) m->rot.stop_worker();
    PlanDeleter<b2s_mixer>()(m);
}

// `let mut osc = Complex32::new(1.0, 0.0)` (receive.rs:58, :73; transmit.rs:101)
int32_t b2s_mixer_reset(b2s_mixer *m) {
    if (!m) return b2s_fail(nullptr, B2S_EINVAL, "mixer is NULL");
    return replay_reset(&m->rot);
}

// ≙ Apply::work (apply.rs:100-131) over one of the closures: m = min(n_in, n_out_cap) samples (:109)
int32_t b2s_mixer_exec(b2s_mixer *m, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                       size_t *consumed, size_t *produced) {
    if (!m || !consumed || !produced) return b2s_fail(m ? m->ctx : nullptr, B2S_EINVAL, "b2s_mixer_exec: NULL argument");
    const size_t n = std::min(n_in, n_out_cap);
    *consumed = n; *produced = n;
    if (n == 0) return B2S_OK;
    if (!d_in || !d_out) return b2s_fail(m->ctx, B2S_EINVAL, "b2s_mixer_exec: NULL buffer");
    const bool weaver = m->op == B2S_MIX_WEAVER_F32;
    const size_t ob = weaver ? sizeof(float) : sizeof(float2);
    if (((uintptr_t)d_in & 7) || ((uintptr_t)d_out & (ob - 1)))
        return b2s_fail(m->ctx, B2S_EINVAL, "b2s_mixer_exec: a slice is not aligned to its item");
    // a thread reads in[s] and writes out[s]: the ROTATE ops may run exactly in place; the Weaver's f32 out[s] lies on
    // in[s / 2], which another thread reads, so it needs disjoint slices
    if (weaver ? overlap(d_in, n * sizeof(float2), d_out, n * ob)
               : bad_alias(d_out, n * ob, ob, d_in, n * sizeof(float2), sizeof(float2)))
        return b2s_fail(m->ctx, B2S_EINVAL, "b2s_mixer_exec: input and output overlap");
    NvtxRange nvtx("b2s_mixer_exec");
    const float2 *in = (const float2 *)d_in;
    switch (m->op) {
        case B2S_MIX_ROTATE_C32: return replay_exec(&m->rot, in, (float2 *)d_out, n, EpiRotate{});
        case B2S_MIX_ROTATE_SCALE_C32: return replay_exec(&m->rot, in, (float2 *)d_out, n, EpiRotateScale{m->param});
        case B2S_MIX_WEAVER_F32: return replay_exec(&m->rot, in, (float *)d_out, n, EpiWeaver{m->param});
    }
    return b2s_fail(m->ctx, B2S_EINVAL, "b2s_mixer_exec: bad op");
}

// bpf[i] = Complex32::from_polar(1.0, i as f32 * TAU * offset / sample_rate) * tap[i]   (xlating_fir.rs:80-86)
// rotator phase increment for the block: -TAU * offset * decimation as f32 / sample_rate        (:97-99)
int32_t b2s_xlating_taps(const float *taps, size_t ntaps, float offset, float sample_rate, size_t decimation,
                         float *bpf_interleaved, float *rotator_phase_incr) {
    if (!taps || !bpf_interleaved || !rotator_phase_incr || decimation == 0)
        return b2s_fail(nullptr, B2S_EINVAL, "b2s_xlating_taps: bad argument");
    const float TAU = 6.28318530717958647692f;
    for (size_t i = 0; i < ntaps; i++) {
        const float th = (float)i * TAU * offset / sample_rate;
        bpf_interleaved[2 * i] = (1.0f * std::cos(th)) * taps[i];
        bpf_interleaved[2 * i + 1] = (1.0f * std::sin(th)) * taps[i];
    }
    *rotator_phase_incr = -TAU * offset * (float)decimation / sample_rate;
    return B2S_OK;
}

}  // extern "C"
