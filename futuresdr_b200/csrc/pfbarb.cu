// pfbarb.cu -- polyphase arbitrary-rate resampler (src/blocks/pfb/arb_resampler.rs:90-231,
// pfb/utilities.rs:5-25, pfb/window_buffer.rs:13-44) on the device.
//
// The reference is a strictly sequential state machine: a f32 timing recurrence
// (update_timing_state :132-140, `tau -= 1.0` :184-186) decides, sample by sample, how many
// outputs are produced and which two polyphase arms are blended.  The recurrence does not
// depend on the data, only on (rate, num_filters, number of samples), so it is split off:
//   * host: replays the reference's f32 recurrence once per call, bit-for-bit (plain C float
//     ops, no contraction), and records the timing state at the start of every 32-sample
//     sub-block -- 16 bytes per 32 samples, this is what makes output COUNTS and arm indices
//     identical to the reference;
//   * device: every sub-block is replayed by one thread from its recorded state (same IEEE
//     operations via __fadd_rn/__fmul_rn), which yields one descriptor per output in shared
//     memory; then all threads of the CTA evaluate the outputs: two T-tap dot products on the
//     window ending at the right sample, blended with (1-mu, mu) (:159-176, Boundary :147-156).
// PERIODIC SCHEDULE (round 2): the timing state (tau, mu, base_index, state) is a deterministic map on a finite set
// of f32 values, and the whole trajectory starts from tau = 0, so it is a pure cycle: Brent's algorithm finds its
// length at plan time (2-13 M input samples for the rates tried, < 0.1 s), the state at every 8th sample of ONE period
// is uploaded once (16 bytes per record), and a call only needs its position in the cycle: no per-call host replay,
// no per-call record upload, output counts still bit-identical.  Rates whose trajectory has a pre-period or a cycle
// longer than 2^25 samples keep the per-call host replay above.
// The input history (the reference's WindowBuffer) is the shared window buffer of pfb_common.cuh
// with one window, carried between calls, including the scattered start-up fill.
#include <cmath>
#include <cstdlib>

#include "pfb_common.cuh"

namespace {
constexpr int kSB = 32;            // input samples per recorded sub-block
constexpr int kPaThreads = 256;
constexpr int kDescCap = 4096;     // outputs per CTA (descriptor slots in shared memory)
constexpr int kPaSmemMax = 3 * kDescCap * 4 + 2 * 64 * 1024;   // descriptors + input tile + arms

struct SubRec {                    // timing state at a sub-block boundary
    uint32_t out0;                 // index (within the call) of the sub-block's first output
    float tau;
    float mu;
    uint32_t base_flag;            // base_index | boundary << 31
};
}  // namespace

struct b2s_pfbarb {
    b2s_ctx *ctx = nullptr;
    size_t num_filters = 0, T = 0, ntaps = 0;
    float rate = 1.f, delay = 1.f;
    Buf<float2> d_arms;            // [num_filters][T] PAIRS (arm_b[T-1-j], arm_{(b+1) % N}[T-1-j]), time-reversed: an output blends
                                   // arm b and its successor (arm 0 after the last one: the Boundary state), one 8-byte load per tap
    PfbWindows win;                // one window of T samples: the input history
    // State (host): arb_resampler.rs:40-52
    float tau = 0.f, bf = 0.f, mu = 0.f;
    size_t base_index = 0;
    bool boundary = false;
    // periodic schedule (plan time): records at every kPerSB-th sample of one period, outputs per period
    bool periodic = false;
    uint64_t lambda = 0, out_per_period = 0, gpos = 0;   // gpos: samples processed since the window filled
    std::vector<SubRec> tab;       // host copy, tab[j] = state before sample kPerSB*j of the period (out0 = outputs so far)
    Buf<SubRec> d_tab;
    // per-call records
    Buf<SubRec, Mem::Pinned> h_recs;
    Buf<SubRec> d_recs;
};

namespace {

// `bf.floor() as usize` (arb_resampler.rs:136): Rust's float -> integer cast saturates -- negative and NaN give 0.  With
// rate > num_filters, tau is still negative when the output after a Boundary state advances it, so bf < 0 does occur; a
// plain C cast of a negative float to an unsigned type is undefined (it wraps to 0xFFFFFFFF on x86-64) and would stop
// the timing loop for good.
__host__ __device__ __forceinline__ uint32_t pfb_arm_index(float bf) {
    const float f = floorf(bf);
    return f > 0.f ? (f < 4294967296.f ? (uint32_t)f : 0xffffffffu) : 0u;
}

// Outputs one input sample can produce, at most.  A sample starts with tau >= -1/N (tau >= (N-1)/N when the Boundary
// state is entered, then tau -= 1) and emits one output per step of `delay` until tau >= 1: at most
// ceil(rate * (1 + 1/N)) outputs.  For rate <= N that is ceil(rate) + 1; above it, 2 more for f32 rounding.
inline size_t pfbarb_per_sample_max(float rate, size_t num_filters) {
    if (rate <= (float)num_filters) return (size_t)std::ceil(rate) + 1;
    return (size_t)std::ceil((double)rate * (1.0 + 1.0 / (double)num_filters)) + 2;
}

__device__ __forceinline__ float2 pfb_x(const float2 *__restrict__ hist, const float2 *__restrict__ in, int L,
                                        long long idx) {
    return idx < L ? hist[idx] : __ldg(in + (idx - L));
}

struct PaParams {
    const float2 *in, *hist;
    float2 *out;
    const float2 *arms;            // [N][T] pairs (arm b, arm b+1)
    const SubRec *recs;            // periodic: the plan's table; otherwise this call's records
    long long n_in, nsub, nout;
    int sub_per_cta, N, T, sb_len;
    float delay;
    int arms_in_smem, tile_in_smem, tile_cap;
    // periodic schedule: sub-block i of the call is sub-block (lsb_first + i) of the unrolled cycle
    int periodic;
    unsigned long long lambda, out_per_period, R, g0, lsb_first;
    long long O_g0;                // outputs the cycle has produced before sample g0
};

struct SubStart { float tau, mu; uint32_t base_flag; long long s_beg, s_end, o_start; };

__device__ __forceinline__ SubStart pfb_sub_start(const PaParams &P, long long i) {
    SubStart r;
    if (P.periodic) {
        const unsigned long long lsb = P.lsb_first + (unsigned long long)i;
        const unsigned long long k = lsb / P.R, j = lsb - k * P.R;
        const SubRec rec = P.recs[j];
        const unsigned long long gs = k * P.lambda + j * (unsigned long long)P.sb_len;
        const unsigned long long ge = min(gs + (unsigned long long)P.sb_len, (k + 1) * P.lambda);
        r.tau = rec.tau; r.mu = rec.mu; r.base_flag = rec.base_flag;
        r.s_beg = (long long)gs - (long long)P.g0;
        r.s_end = min((long long)ge - (long long)P.g0, P.n_in);
        r.o_start = (long long)(k * P.out_per_period + rec.out0) - P.O_g0;
    } else {
        const SubRec rec = P.recs[i];
        r.tau = rec.tau; r.mu = rec.mu; r.base_flag = rec.base_flag;
        r.s_beg = i * P.sb_len;
        r.s_end = min(r.s_beg + P.sb_len, P.n_in);
        r.o_start = rec.out0;
    }
    return r;
}

__global__ void __launch_bounds__(kPaThreads) pfb_kernel(const PaParams P) {
    extern __shared__ __align__(16) unsigned char psm[];
    uint32_t *d_s1 = reinterpret_cast<uint32_t *>(psm);          // window start of y1 | boundary << 31
    uint32_t *d_b0 = d_s1 + kDescCap;                            // arm of y0
    float *d_mu = reinterpret_cast<float *>(d_b0 + kDescCap);
    float2 *s_x = reinterpret_cast<float2 *>(d_mu + kDescCap);   // the CTA's span of [hist | in]
    float2 *s_arms = s_x + (P.tile_in_smem ? P.tile_cap : 0);
    const int N = P.N, T = P.T;

    const long long sb0 = (long long)blockIdx.x * P.sub_per_cta;
    const long long sb1 = min(sb0 + P.sub_per_cta, P.nsub);
    const SubStart first = pfb_sub_start(P, sb0);
    const long long o_first = max(first.o_start, 0ll);
    const long long o_end = sb1 == P.nsub ? P.nout : pfb_sub_start(P, sb1).o_start;
    const long long s_lo = max(first.s_beg, 0ll);                // first sample of the CTA (call coordinates)
    const long long s_hi = pfb_sub_start(P, sb1 - 1).s_end;
    // arm rows in shared memory with an ODD row stride: the threads of a warp read different arms at the same tap
    // index, and with a stride of 16 all 32 of them would hit two banks.
    // In shared memory the table is PLANAR (one float row per arm, arm b+1 is the second row a thread reads) with an odd
    // row stride: a 4-byte access has 32 banks for the 32 lanes, so any set of arms is conflict-free at a given tap index
    // -- 8-byte pair rows would have 16 bank pairs for 32 arms and take two passes per load.
    const int TS = P.arms_in_smem ? (T | 1) : T;
    float *s_tap = reinterpret_cast<float *>(s_arms);
    if (P.arms_in_smem)
        for (int j = threadIdx.x; j < N * T; j += kPaThreads) s_tap[(j / T) * TS + (j % T)] = P.arms[j].x;
    if (P.tile_in_smem) {
        // the outputs of sample s read [hist | in][s+1 .. s+T] (Boundary: [s .. s+T-1] as well), s in [s_lo, s_hi):
        // items s_lo .. s_hi+T-1.  (One more would read in[n_in]: compute-sanitizer caught exactly that.)
        const int cnt = (int)(s_hi - s_lo) + T;
        for (int j = threadIdx.x; j < cnt; j += kPaThreads) s_x[j] = pfb_x(P.hist, P.in, T, s_lo + j);
    }

    // ---- phase 1: replay the timing recurrence of each sub-block (one thread per sub-block)
    for (long long sb = sb0 + threadIdx.x; sb < sb1; sb += kPaThreads) {
        const SubStart r = pfb_sub_start(P, sb);
        float tau = r.tau, mu = r.mu;
        uint32_t base = r.base_flag & 0x7fffffffu;
        bool boundary = (r.base_flag >> 31) != 0;
        long long o = r.o_start - o_first;                        // < 0 while replaying samples in front of the call
        const float fN = (float)N, delay = P.delay;
        for (long long s = r.s_beg; s < r.s_end; s++) {
            while (base < (uint32_t)N) {
                if (boundary) {
                    if (s >= 0) { d_s1[o] = (uint32_t)(s + 1 - s_lo) | 0x80000000u; d_b0[o] = (uint32_t)(N - 1); d_mu[o] = mu; }
                    o++;
                    tau = __fadd_rn(tau, delay);
                    const float bf = __fmul_rn(tau, fN);
                    base = pfb_arm_index(bf);
                    mu = __fsub_rn(bf, (float)base);
                    boundary = false;
                } else if (base == (uint32_t)(N - 1)) {
                    boundary = true;
                    base = (uint32_t)N;
                } else {
                    if (s >= 0) { d_s1[o] = (uint32_t)(s + 1 - s_lo); d_b0[o] = base; d_mu[o] = mu; }
                    o++;
                    tau = __fadd_rn(tau, delay);
                    const float bf = __fmul_rn(tau, fN);
                    base = pfb_arm_index(bf);
                    mu = __fsub_rn(bf, (float)base);
                }
            }
            tau = __fsub_rn(tau, 1.0f);
            base -= (uint32_t)N;
        }
    }
    __syncthreads();

    // ---- phase 2: evaluate the outputs.  y0 = arm b0, y1 = arm b0+1 on the same window (Interpolate), or arm N-1 on the
    // previous window and arm 0 on the current one (Boundary): per tap ONE 8-byte sample load and ONE 8-byte tap-pair load
    const float2 *A = P.arms;                                    // pair rows in global memory (tables too large for smem)
    const uint32_t cnt = (uint32_t)(o_end - o_first);
    for (uint32_t o = threadIdx.x; o < cnt; o += kPaThreads) {
        const uint32_t w = d_s1[o];
        const bool boundary = (w >> 31) != 0;
        const int s1 = (int)(w & 0x7fffffffu);                   // relative to s_lo
        const uint32_t b0 = d_b0[o];
        const float mu = d_mu[o];
        const float2 *pr = A + (size_t)b0 * T;
        float2 y0 = make_float2(0.f, 0.f), y1 = make_float2(0.f, 0.f);
        if (P.tile_in_smem && P.arms_in_smem) {
            const float *t0 = s_tap + b0 * TS, *t1 = s_tap + (b0 + 1 == (uint32_t)N ? 0u : b0 + 1) * TS;
            const float2 *xb = s_x + s1;
            if (!boundary) {
#pragma unroll 4
                for (int j = 0; j < T; j++) {
                    const float2 v = xb[j];
                    const float ta = t0[j], tb = t1[j];
                    y0.x = fmaf(v.x, ta, y0.x); y0.y = fmaf(v.y, ta, y0.y);
                    y1.x = fmaf(v.x, tb, y1.x); y1.y = fmaf(v.y, tb, y1.y);
                }
            } else {
                const float2 *xa = xb - 1;
                for (int j = 0; j < T; j++) {
                    const float2 va = xa[j], vb = xb[j];
                    const float ta = t0[j], tb = t1[j];
                    y0.x = fmaf(va.x, ta, y0.x); y0.y = fmaf(va.y, ta, y0.y);
                    y1.x = fmaf(vb.x, tb, y1.x); y1.y = fmaf(vb.y, tb, y1.y);
                }
            }
        } else if (P.tile_in_smem) {
            const float2 *xb = s_x + s1;
            if (!boundary) {
#pragma unroll 4
                for (int j = 0; j < T; j++) {
                    const float2 v = xb[j], t = pr[j];
                    y0.x = fmaf(v.x, t.x, y0.x); y0.y = fmaf(v.y, t.x, y0.y);
                    y1.x = fmaf(v.x, t.y, y1.x); y1.y = fmaf(v.y, t.y, y1.y);
                }
            } else {
                const float2 *xa = xb - 1;
                for (int j = 0; j < T; j++) {
                    const float2 va = xa[j], vb = xb[j], t = pr[j];
                    y0.x = fmaf(va.x, t.x, y0.x); y0.y = fmaf(va.y, t.x, y0.y);
                    y1.x = fmaf(vb.x, t.y, y1.x); y1.y = fmaf(vb.y, t.y, y1.y);
                }
            }
        } else {
            const int s0 = boundary ? s1 - 1 : s1;
            for (int j = 0; j < T; j++) {
                const float2 va = pfb_x(P.hist, P.in, T, s_lo + s0 + j), vb = pfb_x(P.hist, P.in, T, s_lo + s1 + j);
                const float2 t = pr[j];
                y0.x = fmaf(va.x, t.x, y0.x); y0.y = fmaf(va.y, t.x, y0.y);
                y1.x = fmaf(vb.x, t.y, y1.x); y1.y = fmaf(vb.y, t.y, y1.y);
            }
        }
        // (1.0 - mu) * buff[0] + mu * buff[1]   (arb_resampler.rs:153,:176)
        const float a = __fsub_rn(1.0f, mu);
        float2 r;
        r.x = __fadd_rn(__fmul_rn(a, y0.x), __fmul_rn(mu, y1.x));
        r.y = __fadd_rn(__fmul_rn(a, y0.y), __fmul_rn(mu, y1.y));
        P.out[(size_t)o_first + o] = r;
    }
}

// The reference's timing state machine on the host (State::consume_single's control flow,
// arb_resampler.rs:142-188), one input sample per step().  Plain float locals: the host side of this file is
// built by g++ for x86-64 without -ffast-math / contraction, so every + and * is one IEEE binary32 SSE
// operation and the sequence is the reference's.  (`bf` is never read before it is overwritten, so it is
// not part of the state.)
struct Timing {
    float tau = 0.f, mu = 0.f;
    uint32_t base = 0;
    bool boundary = false;
    bool operator==(const Timing &o) const { return tau == o.tau && mu == o.mu && base == o.base && boundary == o.boundary; }
    inline uint32_t step(uint32_t N, float fN, float delay) {     // returns the outputs this sample produced
        uint32_t o = 0;
        while (base < N) {
            if (boundary) {
                o++;
                tau = tau + delay; const float bf = tau * fN; base = pfb_arm_index(bf); mu = bf - (float)base;
                boundary = false;
            } else if (base == N - 1) {
                boundary = true;
                base = N;
            } else {
                o++;
                tau = tau + delay; const float bf = tau * fN; base = pfb_arm_index(bf); mu = bf - (float)base;
            }
        }
        tau = tau - 1.0f;
        base -= N;
        return o;
    }
    SubRec rec(uint32_t out0) const { return SubRec{out0, tau, mu, base | (boundary ? 0x80000000u : 0u)}; }
};

constexpr int kPerSB = 8;                      // samples per record of the periodic table
constexpr uint64_t kMaxPeriod = 1ull << 25;    // 64 MiB of records at most

// Brent's cycle detection on the per-sample map, then one replay of the period to build the table.
bool build_periodic_schedule(b2s_pfbarb *p) {
    const uint32_t N = (uint32_t)p->num_filters;
    const float fN = (float)N, delay = p->delay;
    Timing tort, hare;
    uint64_t power = 1, lam = 1;
    hare.step(N, fN, delay);
    while (!(tort == hare)) {
        if (power == lam) {
            if (power > kMaxPeriod) return false;
            tort = hare; power *= 2; lam = 0;
        }
        hare.step(N, fN, delay);
        lam++;
    }
    if (lam > kMaxPeriod) return false;
    const uint64_t R = ceil_div((size_t)lam, (size_t)kPerSB);
    std::vector<SubRec> tab(R);
    Timing t;
    uint64_t o = 0;
    for (uint64_t s = 0; s < lam; s++) {
        if ((s % kPerSB) == 0) tab[s / kPerSB] = t.rec((uint32_t)o);
        o += t.step(N, fN, delay);
        if (o >= (1ull << 32)) return false;
    }
    if (!(t == Timing())) return false;        // a pre-period: the start state is not on the cycle
    p->tab.swap(tab);
    p->lambda = lam; p->out_per_period = o;
    return true;
}

// outputs the cycle has produced before its sample c (0 <= c <= lambda)
uint64_t outputs_before(const b2s_pfbarb *p, uint64_t c) {
    if (c >= p->lambda) return p->out_per_period + outputs_before(p, c - p->lambda);
    const uint64_t j = c / kPerSB;
    const SubRec &r = p->tab[j];
    Timing t;
    t.tau = r.tau; t.mu = r.mu; t.base = r.base_flag & 0x7fffffffu; t.boundary = (r.base_flag >> 31) != 0;
    uint64_t o = r.out0;
    const uint32_t N = (uint32_t)p->num_filters;
    for (uint64_t s = j * kPerSB; s < c; s++) o += t.step(N, (float)N, p->delay);
    return o;
}

}  // namespace

extern "C" {

// Host-only: the period of the timing recurrence (what the plan's table covers).  No device needed.
int32_t b2s_pfbarb_period(float rate, size_t num_filters, uint64_t *period_items, uint64_t *outputs_per_period) {
    if (!(rate > 0.f) || num_filters == 0 || !period_items || !outputs_per_period)
        return b2s_fail(nullptr, B2S_EINVAL, "b2s_pfbarb_period: bad argument");
    b2s_pfbarb tmp;
    tmp.num_filters = num_filters; tmp.rate = rate; tmp.delay = 1.0f / rate;
    const bool ok = build_periodic_schedule(&tmp);
    *period_items = ok ? tmp.lambda : 0;
    *outputs_per_period = ok ? tmp.out_per_period : 0;
    return B2S_OK;
}

int32_t b2s_pfbarb_plan_c32(b2s_ctx *ctx, const float *taps, size_t ntaps, size_t num_filters, float rate,
                            b2s_pfbarb **out) {
    if (!ctx || !out || !taps) return b2s_fail(ctx, B2S_EINVAL, "b2s_pfbarb_plan_c32: NULL argument");
    *out = nullptr;
    // the reference asserts these (arb_resampler.rs:92-104)
    if (!(rate > 0.f)) return b2s_fail(ctx, B2S_EINVAL, "PfbArbResampler: resampling rate must be greater than zero");
    if (num_filters == 0) return b2s_fail(ctx, B2S_EINVAL, "PfbArbResampler: number of filter banks must be greater than zero");
    if (ntaps < num_filters) return b2s_fail(ctx, B2S_EINVAL, "PfbArbResampler: prototype filter length must be at least num_filters");
    // a 32-sample sub-block must fit the descriptor tile of a CTA: pfbarb_per_sample_max * 32 <= kDescCap (rate <= 126
    // with at least as many arms as the rate, less above it)
    if (num_filters > (1u << 20) || rate > 126.f || pfbarb_per_sample_max(rate, num_filters) * kSB > (size_t)kDescCap)
        return b2s_fail(ctx, B2S_EUNSUPPORTED, "PfbArbResampler: rate %f too large for %zu arms (a sample may produce more outputs than one CTA holds)", (double)rate, num_filters);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_pfbarb> p(new b2s_pfbarb());
    p->ctx = ctx; p->num_filters = num_filters; p->ntaps = ntaps; p->rate = rate;
    p->delay = 1.0f / rate;
    std::vector<float> arms;
    const size_t T = pfb_partition(taps, ntaps, num_filters, arms);
    p->T = T;
    std::vector<float2> pairs(num_filters * T);      // time-reversed
    for (size_t b = 0; b < num_filters; b++)
        for (size_t j = 0; j < T; j++)
            pairs[b * T + j] = make_float2(arms[b * T + T - 1 - j], arms[((b + 1) % num_filters) * T + T - 1 - j]);
    B2S_TRY(p->d_arms.upload(ctx, pairs.data(), pairs.size(), "pfbarb arms"));
    B2S_TRY(p->win.init(ctx, 1, (int)T, false, "pfbarb history"));
    p->periodic = getenv("B2S_PFBARB_NO_PERIODIC") ? false : build_periodic_schedule(p.get());
    if (p->periodic) B2S_TRY(p->d_tab.upload(ctx, p->tab.data(), p->tab.size(), "pfbarb schedule table"));
    B2S_TRY(smem_optin<pfb_kernel>(ctx, kPaSmemMax));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    B2S_TRY(b2s_pfbarb_reset(p.get()));
    *out = p.release();
    return B2S_OK;
}

void b2s_pfbarb_destroy(b2s_pfbarb *p) { PlanDeleter<b2s_pfbarb>()(p); }

int32_t b2s_pfbarb_reset(b2s_pfbarb *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "pfbarb is NULL");
    DeviceGuard g(p->ctx->device);
    p->tau = 0.f; p->bf = 0.f; p->mu = 0.f; p->base_index = 0; p->boundary = false;
    p->gpos = 0;
    return p->win.reset(p->ctx);                                   // WindowBuffer::new(len, pad_start=false)
}

int32_t b2s_pfbarb_exec(b2s_pfbarb *p, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                        size_t *consumed, size_t *produced, int32_t *call_again) {
    if (!p || !consumed || !produced || !call_again) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_pfbarb_exec: NULL argument");
    b2s_ctx *ctx = p->ctx;
    *consumed = 0; *produced = 0; *call_again = 0;
    DeviceGuard g(ctx->device);
    const int T = (int)p->T;
    const float2 *in = (const float2 *)d_in;
    // fill filter history (arb_resampler.rs:199-215)
    if (!p->win.full()) {
        const size_t c = std::min(p->win.missing(), n_in);
        B2S_TRY(p->win.push(ctx, in, c));
        *consumed = c;
        if (n_in - c > 0) *call_again = 1;
        return B2S_OK;
    }
    // nitem_to_process = min(ninput_items, (noutput_items as f32 / rate) as usize)   (:218)
    const size_t cap = (size_t)((float)n_out_cap / p->rate);
    const size_t n = std::min(n_in, cap);
    if (n == 0) return B2S_OK;
    if (!d_in || !d_out) return b2s_fail(ctx, B2S_EINVAL, "b2s_pfbarb_exec: NULL buffer");
    if (n >= (1ull << 31)) return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_pfbarb_exec: more than 2^31 items per call");
    NvtxRange nvtx("b2s_pfbarb_exec");
    PaParams P{};
    P.in = in; P.hist = p->win.hist.get(); P.out = (float2 *)d_out; P.arms = p->d_arms.get();
    P.n_in = (long long)n; P.N = (int)p->num_filters; P.T = T; P.delay = p->delay;
    size_t nout;
    Timing after;                                  // fallback path: the state to commit once the call is accepted
    if (p->periodic) {
        // position in the cycle -> output count and the sub-blocks of the table this call touches: O(1) host work
        const uint64_t g0 = p->gpos, g1 = g0 + n, lam = p->lambda, R = p->tab.size();
        const uint64_t O0 = outputs_before(p, g0);
        const uint64_t O1 = (g1 / lam) * p->out_per_period + outputs_before(p, g1 % lam);
        nout = (size_t)(O1 - O0);
        if (nout > n_out_cap)
            return b2s_fail(ctx, B2S_ESTATE, "pfbarb: schedule produces %zu > capacity %zu (the reference would overrun its slice)", nout, n_out_cap);
        const uint64_t lsb_first = g0 / kPerSB;                                   // g0 < lambda
        const uint64_t gl = g1 - 1, lsb_last = (gl / lam) * R + (gl % lam) / kPerSB;
        P.periodic = 1; P.recs = p->d_tab.get(); P.sb_len = kPerSB;
        P.lambda = lam; P.out_per_period = p->out_per_period; P.R = R; P.g0 = g0; P.lsb_first = lsb_first;
        P.O_g0 = (long long)O0;
        P.nsub = (long long)(lsb_last - lsb_first + 1);
    } else {
        // per-call host replay (trajectories with a pre-period / very long cycles): the state at every 32nd sample
        const size_t nsub = ceil_div(n, (size_t)kSB);
        B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));        // the pinned records of the previous call may still be in flight
        if (std::min(p->d_recs.size(), p->h_recs.size()) < nsub + 1) {
            const size_t want = (nsub + 1) * 5 / 4 + 16;
            B2S_TRY(p->d_recs.reserve(ctx, want, "pfbarb records"));
            B2S_TRY(p->h_recs.reserve(ctx, want, "pfbarb pinned records"));
        }
        Timing t;                                  // replay on a COPY: nothing is committed if the call is refused
        t.tau = p->tau; t.mu = p->mu; t.base = (uint32_t)p->base_index; t.boundary = p->boundary;
        const uint32_t N = (uint32_t)p->num_filters;
        uint64_t o = 0;
        for (size_t s = 0; s < n; s++) {
            if ((s % kSB) == 0) p->h_recs.get()[s / kSB] = t.rec((uint32_t)o);
            o += t.step(N, (float)N, p->delay);
        }
        p->h_recs.get()[nsub] = t.rec((uint32_t)o);
        nout = (size_t)o;
        if (nout > n_out_cap || o >= (1ull << 32))
            return b2s_fail(ctx, B2S_ESTATE, "pfbarb: schedule produces %zu > capacity %zu (the reference would overrun its slice)", nout, n_out_cap);
        after = t;
        B2S_CUDA(ctx, cudaMemcpyAsync(p->d_recs.get(), p->h_recs.get(), (nsub + 1) * sizeof(SubRec), cudaMemcpyHostToDevice, ctx->stream));
        P.periodic = 0; P.recs = p->d_recs.get(); P.sb_len = kSB; P.nsub = (long long)nsub;
    }
    P.nout = (long long)nout;
    // CTA tiling: sub-blocks per CTA so that a CTA never exceeds kDescCap outputs
    const size_t per_sample_max = pfbarb_per_sample_max(p->rate, p->num_filters);
    size_t sub_per_cta = kDescCap / (per_sample_max * P.sb_len);
    if (sub_per_cta == 0) return b2s_fail(ctx, B2S_EUNSUPPORTED, "pfbarb: rate %f too high for the descriptor tile", (double)p->rate);
    sub_per_cta = std::min<size_t>(sub_per_cta, kPaThreads);
    P.sub_per_cta = (int)sub_per_cta;
    const unsigned grid = (unsigned)ceil_div((size_t)P.nsub, sub_per_cta);
    const size_t tile_items = sub_per_cta * P.sb_len + p->T + 2;
    P.tile_in_smem = tile_items * sizeof(float2) <= 64 * 1024;
    P.tile_cap = (int)tile_items;
    const size_t arms_smem_bytes = p->num_filters * (p->T | 1) * sizeof(float);        // planar rows, odd stride
    P.arms_in_smem = arms_smem_bytes <= 64 * 1024;
    const size_t smem = 3 * kDescCap * sizeof(uint32_t) + (P.tile_in_smem ? tile_items * sizeof(float2) : 0) +
                        (P.arms_in_smem ? arms_smem_bytes : 0);
    pfb_kernel<<<grid, kPaThreads, smem, ctx->stream>>>(P);
    B2S_CHECK_LAUNCH(ctx);
    B2S_TRY(p->win.slide(ctx, in, 0, (long long)n));
    // the call is on the stream: commit the timing state
    if (p->periodic) p->gpos = (p->gpos + n) % p->lambda;
    else { p->tau = after.tau; p->mu = after.mu; p->base_index = after.base; p->boundary = after.boundary; }
    *consumed = n; *produced = nout;
    return B2S_OK;
}

}  // extern "C"
