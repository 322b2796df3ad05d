// mavg.cu -- MovingAvg<WIDTH> (src/blocks/moving_avg.rs:24-116), the tail of the spectrum pipe
// (examples/spectrum/src/bin/cpu.rs:21-28: Fft(shift) -> |x|^2 -> MovingAvg -> sink): SURVEY §8f-3.
//
// Per bin i an exponential average over consecutive WIDTH-item chunks:
//     avg[i] = (1 - decay) * avg[i] + decay * t        (t finite)      (:87)
//     avg[i] *= 1 - decay                              (t not finite)  (:89)
// and every `history_size` chunks the WIDTH averages are emitted (:95-99).  The recurrence is
// sequential over chunks but independent across bins: one thread per bin walks the chunks in order
// with un-fused IEEE multiplies/adds (identical to the reference bit for bit), reads are coalesced
// across bins.  The state (avg[], chunk counter) lives on the device between calls.
#include <cmath>

#include "common.cuh"

struct b2s_mavg {
    b2s_ctx *ctx = nullptr;
    size_t width = 0, history = 1;
    float decay = 0.1f;
    Buf<float> d_avg;
    size_t i = 0;                 // chunks since the last emission (host mirror; data-independent)
};

namespace {

// A CTA owns 32 bins.  The recurrence itself is 2 dependent operations per chunk in ONE lane per bin
// (warp 0), which cannot keep HBM busy on its own, so all 8 warps stream blocks of 64 chunks (64 rows of
// 128 bytes) into a 4-deep shared-memory ring with cp.async (LDGSTS: no registers held across the wait),
// three blocks ahead of the one warp 0 is walking.  Operations and their order are the reference's
// (un-fused IEEE mul/add).  (A register double buffer, one block ahead, waits a whole DRAM round trip
// per block.)
constexpr int kMaBins = 32, kMaFrames = 64, kMaWarps = 8, kMaStages = 4;

__global__ void __launch_bounds__(32 * kMaWarps)
mavg_kernel(const float *__restrict__ in, float *__restrict__ out, float *avg, int width,
            long long nchunks, int history, int i0, float decay, long long max_out) {
    __shared__ float buf[kMaStages][kMaFrames][kMaBins];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.x * kMaBins + lane;
    const bool live = b < width;
    const long long nblk = (nchunks + kMaFrames - 1) / kMaFrames;
    constexpr int PER = kMaFrames / kMaWarps;            // rows each warp fetches per block
    auto issue = [&](long long blk) {                    // always commits a group, possibly empty
        if (blk < nblk) {
            const int stage = (int)(blk % kMaStages);
#pragma unroll
            for (int k = 0; k < PER; k++) {
                const int f = warp + k * kMaWarps;
                const long long c = blk * kMaFrames + f;
                const bool ok = live && c < nchunks;
                cp_async::ca4(&buf[stage][f][lane], ok ? in + c * width + b : in, ok);
            }
        }
        cp_async::commit();
    };
    float a = live ? avg[b] : 0.0f;
    const float keep = __fsub_rn(1.0f, decay);
    int i = i0;
    long long produced = 0;
    float *outp = out + (live ? b : 0);                  // next emission of this bin (only warp 0 uses it)
    for (int s = 0; s < kMaStages - 1; s++) issue(s);
    for (long long blk = 0; blk < nblk; blk++) {
        issue(blk + kMaStages - 1);                      // refills the stage warp 0 finished in the previous iteration
        cp_async::wait<kMaStages - 1>();
        __syncthreads();                                 // block blk has landed for every thread's copies
        if (warp == 0 && live) {
            const int stage = (int)(blk % kMaStages);
            const int nf = (int)min((long long)kMaFrames, nchunks - blk * kMaFrames);
            // One warp walks the chunks in order, so what matters is the length of the per-chunk instruction
            // sequence: branch-free body (selects and a predicated store), loads and decay*t products hoisted
            // out of the dependent chain, a running output pointer instead of a 64-bit multiply.
            auto step = [&](float t, float dt) {
                const float ka = __fmul_rn(keep, a);              // == a * keep of the non-finite branch (:89)
                a = isfinite(t) ? __fadd_rn(ka, dt) : ka;
                const bool emit = ++i == history;
                if (emit && produced < max_out) *outp = a;
                outp += emit ? width : 0;
                produced += emit ? 1 : 0;
                i = emit ? 0 : i;
            };
            if (nf == kMaFrames) {
#pragma unroll 1
                for (int f0 = 0; f0 < kMaFrames; f0 += 16) {
                    float t[16], dt[16];
#pragma unroll
                    for (int k = 0; k < 16; k++) { t[k] = buf[stage][f0 + k][lane]; dt[k] = __fmul_rn(decay, t[k]); }
#pragma unroll
                    for (int k = 0; k < 16; k++) step(t[k], dt[k]);
                }
            } else {
                for (int f = 0; f < nf; f++) {
                    const float t = buf[stage][f][lane];
                    step(t, __fmul_rn(decay, t));
                }
            }
        }
        __syncthreads();                                 // stage may be overwritten by the next iteration's issue
    }
    if (warp == 0 && live) avg[b] = a;
}

}  // namespace

extern "C" {

int32_t b2s_mavg_create(b2s_ctx *ctx, size_t width, float decay_factor, size_t history_size, b2s_mavg **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_mavg_create: NULL argument");
    *out = nullptr;
    if (width == 0 || history_size == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_mavg_create: width and history_size must be > 0");
    if (!(decay_factor >= 0.0f && decay_factor <= 1.0f))                        // moving_avg.rs:58-61
        return b2s_fail(ctx, B2S_EINVAL, "decay_factor must be in [0, 1]");
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_mavg> m(new b2s_mavg());
    m->ctx = ctx; m->width = width; m->history = history_size; m->decay = decay_factor;
    B2S_TRY(m->d_avg.alloc(ctx, width, "mavg state"));
    B2S_CUDA(ctx, cudaMemsetAsync(m->d_avg.get(), 0, width * sizeof(float), ctx->stream));
    *out = m.release();
    return B2S_OK;
}

void b2s_mavg_destroy(b2s_mavg *m) { PlanDeleter<b2s_mavg>()(m); }

// One Kernel::work call (moving_avg.rs:72-115).  consumed / produced are in ITEMS (multiples of WIDTH).
int32_t b2s_mavg_exec(b2s_mavg *m, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                      size_t *consumed, size_t *produced) {
    if (!m || !consumed || !produced) return b2s_fail(m ? m->ctx : nullptr, B2S_EINVAL, "b2s_mavg_exec: NULL argument");
    const size_t W = m->width;
    // while (consumed+1)*W <= in.len() && (produced+1)*W <= out.len()   (:82)
    size_t c = 0, p = 0, i = m->i;
    const size_t cin = n_in / W, cout = n_out_cap / W;
    while (c + 1 <= cin && p + 1 <= cout) {
        // jump to the next emission (or to the end of the input)
        const size_t to_emit = m->history - i;
        if (c + to_emit <= cin) { c += to_emit; p += 1; i = 0; }
        else { i += cin - c; c = cin; }
    }
    *consumed = c * W; *produced = p * W;
    if (c == 0) return B2S_OK;
    if (!d_in || (!d_out && p)) return b2s_fail(m->ctx, B2S_EINVAL, "b2s_mavg_exec: NULL buffer");
    DeviceGuard g(m->ctx->device);
    NvtxRange nvtx("b2s_mavg_exec");
    mavg_kernel<<<(unsigned)ceil_div(W, (size_t)kMaBins), 32 * kMaWarps, 0, m->ctx->stream>>>(
        (const float *)d_in, (float *)d_out, m->d_avg.get(), (int)W, (long long)c, (int)m->history, (int)m->i, m->decay,
        (long long)p);
    B2S_CHECK_LAUNCH(m->ctx);
    m->i = i;
    return B2S_OK;
}

}  // extern "C"
