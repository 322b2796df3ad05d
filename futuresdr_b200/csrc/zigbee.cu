// zigbee.cu -- the ZigBee (IEEE 802.15.4 O-QPSK) receiver's ClockRecoveryMm and Decoder (examples/zigbee/src/
// {clock_recovery_mm,decoder}.rs) with the Mac's FCS check (mac.rs:62-85) as device blocks (DESIGN §4.16).  With
// Apply(QuadDemod) and Apply(DcBlockF32) in front they are the receive chain of examples/zigbee/src/bin/rx.rs:66-92, and
// only decoded frames leave the device.
//
// ClockRecoveryMm is a data-dependent f32 recurrence, bit-exact only in order: mm_kernel is one CTA whose lane 0 walks
// the loop while the other warps keep a shared-memory ring of the input filled (cp.async) and flush the outputs.
//
// The Decoder is a state machine over chips (v > 0) whose Search state only asks whether the 32-chip shift register
// matches chip sequence 0, which depends on the stream alone:
//   1. chips_kernel   ballots the chip bits into words and the Search triggers into a bitmap, in parallel.
//   2. walk_kernel    one warp walks from trigger to trigger; in a frame it looks at every 32nd chip only, 32 of them
//                     at a time (one lane each), and applies the transitions in order.
//
// Numerics: __fmul_rn / __fadd_rn / __fsub_rn only and no FTZ, as in the reference's f32.
#include <cmath>
#include <cstdint>

#include "lists.cuh"

namespace {

// ---- ClockRecoveryMm --------------------------------------------------------------------------------------------
constexpr int kMmThreads = 128;        // warp 0: the recurrence (lane 0); warps 1-3: input ring and output flush
constexpr int kMmChunk = 1024;         // ring chunk, in items
constexpr int kMmSlots = 8;            // chunks in the ring
constexpr int kMmRing = kMmChunk * kMmSlots;
constexpr int kMmOut = 1024;           // outputs per phase
constexpr int kWin = 5;                // input items lane 0 holds in registers from ii (a step uses the first two)
constexpr int kFar = 3;                // and the next ones, loaded a step ahead: a fast step moves ii by at most 3

struct MmParams {
    float omega_mid, omega_limit, gain_omega, gain_mu;
    unsigned long long look_ahead;
};
struct MmState {                       // device: the loop's state, and what the last exec did
    float omega, mu, last;
    int err;
    unsigned long long consumed, produced;
};

__device__ __forceinline__ float mm_slice(float x) { return x > 0.0f ? 1.0f : -1.0f; }   // NaN -> -1

// The loop of clock_recovery_mm.rs:74-87 over in[0, n) into out[0, cap).  A phase ends at a barrier: lane 0 runs steps
// while their two input items are in the ring and the phase has output room; meanwhile warps 1-3 flush the previous
// phase's outputs and load the chunks ahead of ii into the slots no step of this phase reads.
__global__ void __launch_bounds__(kMmThreads)
mm_kernel(const float *__restrict__ in, unsigned long long n, float *__restrict__ out, unsigned long long cap,
          MmParams prm, MmState *__restrict__ st) {
    __shared__ float ring[kMmRing];
    __shared__ float ob[2][kMmOut];
    __shared__ unsigned long long sh_ii, sh_oo, sh_lend, sh_cnext;
    __shared__ unsigned sh_pcnt;
    __shared__ int sh_done;
    const int tid = threadIdx.x;
    if (tid == 0) {
        sh_ii = sh_oo = sh_lend = sh_cnext = 0;
        sh_pcnt = 0;
        sh_done = 0;
    }
    float omega = 0.f, mu = 0.f, last = 0.f;
    if (tid == 0) { omega = st->omega; mu = st->mu; last = st->last; }
    const unsigned long long la = prm.look_ahead, nch = (n + kMmChunk - 1) / kMmChunk;
    const unsigned long long run_end = n - la;         // steps run while ii < run_end (the host checks la < n)
    for (int ph = 0;; ph++) {
        __syncthreads();
        const unsigned long long ii0 = sh_ii, oo0 = sh_oo, lend = sh_lend, cnext = sh_cnext;
        const unsigned pcnt = sh_pcnt;
        const int done = sh_done;
        __syncthreads();
        if (done && pcnt == 0) break;
        if (tid == 0) {
            unsigned c = 0;
            if (!done) {
                float *o_s = ob[ph & 1];
                // Indices are relative to ii0 (32-bit) inside a phase.  A step may start while rel < lim: then
                // ii + 1 < lend and ii < run_end.  A step of at most fast_max items is in the slice (n - ii > la).
                const unsigned lend_rel = lend > ii0 ? (unsigned)(lend - ii0) : 0u;
                const unsigned run_rel = run_end > ii0 ? (unsigned)min(run_end - ii0, 0xFFFFFFFFull) : 0u;
                const unsigned lim = min(lend_rel ? lend_rel - 1 : 0u, run_rel);
                const unsigned cmax = (unsigned)min((unsigned long long)kMmOut, cap - oo0);
                const unsigned base = (unsigned)(ii0 % kMmRing);
                const float fast_max = la < 3 ? (float)la : 3.0f;
                // in[ii0 + r], r clamped into the loaded range: the value is only used when r < lend_rel, and the
                // load never touches a slot the loaders are filling (no predicate, one shared address computed once)
                const unsigned ring_s = (unsigned)__cvta_generic_to_shared(ring), rmax = lend_rel ? lend_rel - 1 : 0u;
                auto at = [&](unsigned r) {
                    float v;
                    asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(ring_s + 4u * ((base + min(r, rmax)) % kMmRing)));
                    return v;
                };
                unsigned rel = 0;
                unsigned long long jump = 0;            // a step too long for `rel`: where ii lands
                int err = 0;
                // The window from ii: w[j] = in[ii + j] and d[j] = w[j + 1] - w[j] for j < kWin, and the far end
                // p[k] = in[ii + kWin + k], loaded one step ago.  A fast step first completes the window with p, then
                // shifts it and issues the loads of the next far end, so no load result is used in the step that
                // issues it: the shared-memory latency stays off the chain.
                float w[kWin], d[kWin - 1], p[kFar];
                auto reload = [&]() {
#pragma unroll
                    for (int j = 0; j < kWin; j++) w[j] = at(rel + j);
#pragma unroll
                    for (int j = 0; j + 1 < kWin; j++) d[j] = __fsub_rn(w[j + 1], w[j]);
#pragma unroll
                    for (int k = 0; k < kFar; k++) p[k] = at(rel + kWin + k);
                };
                if (lend_rel) {
                    reload();
                } else {
#pragma unroll
                    for (int j = 0; j < kWin; j++) w[j] = 0.0f;
#pragma unroll
                    for (int j = 0; j + 1 < kWin; j++) d[j] = 0.0f;
#pragma unroll
                    for (int k = 0; k < kFar; k++) p[k] = 0.0f;
                }
                while (rel < lim && c < cmax) {
                    const float o = __fadd_rn(w[0], __fmul_rn(mu, d[0]));
                    const float mm = __fsub_rn(__fmul_rn(mm_slice(last), o), __fmul_rn(mm_slice(o), last));
                    float om = __fadd_rn(omega, __fmul_rn(prm.gain_omega, mm));
                    float dv = __fsub_rn(om, prm.omega_mid);
                    dv = dv < -prm.omega_limit ? -prm.omega_limit : (dv > prm.omega_limit ? prm.omega_limit : dv);  // f32::clamp
                    om = __fadd_rn(prm.omega_mid, dv);
                    const float nmu = __fadd_rn(mu, __fadd_rn(om, __fmul_rn(prm.gain_mu, mm)));
                    const float f = floorf(nmu);
                    if (f <= fast_max) {                // the receiver's steps: selects, no conversion
                        const bool s1 = f >= 1.0f, s2 = f >= 2.0f, s3 = f >= 3.0f;
                        float wx[kWin + kFar], dx[kWin + kFar - 1];
#pragma unroll
                        for (int j = 0; j < kWin; j++) wx[j] = w[j];
#pragma unroll
                        for (int k = 0; k < kFar; k++) wx[kWin + k] = p[k];
#pragma unroll
                        for (int j = 0; j + 1 < kWin; j++) dx[j] = d[j];
#pragma unroll
                        for (int j = kWin - 1; j + 1 < kWin + kFar; j++) dx[j] = __fsub_rn(wx[j + 1], wx[j]);
#pragma unroll
                        for (int j = 0; j < kWin; j++) w[j] = s3 ? wx[j + 3] : s2 ? wx[j + 2] : s1 ? wx[j + 1] : wx[j];
#pragma unroll
                        for (int j = 0; j + 1 < kWin; j++) d[j] = s3 ? dx[j + 3] : s2 ? dx[j + 2] : s1 ? dx[j + 1] : dx[j];
                        rel += (unsigned)s1 + (unsigned)s2 + (unsigned)s3;
#pragma unroll
                        for (int k = 0; k < kFar; k++) p[k] = at(rel + kWin + k);
                    } else {
                        // `as usize` saturates: NaN gives 0; a step past the slice is refused
                        const unsigned long long left = n - (ii0 + rel);
                        if (f > 0.0f && (double)f > (double)left) { err = 1; break; }
                        const unsigned long long step = f > 0.0f ? (unsigned long long)f : 0ull;
                        if (step > kMmRing) {
                            jump = ii0 + rel + step;
                        } else {
                            rel += (unsigned)step;
                            reload();
                        }
                    }
                    o_s[c++] = o;
                    last = o;
                    omega = om;
                    mu = __fsub_rn(nmu, f);
                    if (jump) break;
                }
                const unsigned long long ii = jump ? jump : ii0 + rel, oo = oo0 + c;
                sh_ii = ii;
                sh_oo = oo;
                if (err || !(ii < run_end && oo < cap)) {
                    sh_done = 1;
                    st->omega = omega; st->mu = mu; st->last = last;
                    st->err = err; st->consumed = ii; st->produced = oo;
                }
            }
            sh_pcnt = c;
        } else if (tid >= 32) {
            const int t = tid - 32, nt = kMmThreads - 32;
            const float *o_s = ob[(ph + 1) & 1];        // the previous phase's outputs
            for (unsigned j = t; j < pcnt; j += nt) out[oo0 - pcnt + j] = o_s[j];
            if (!done) {
                // chunks below ii0 / kMmChunk are no longer read: their slots take the chunks up to kMmSlots ahead
                const unsigned long long c_lo = max(cnext, ii0 / kMmChunk);
                const unsigned long long c_hi = min(ii0 / kMmChunk + kMmSlots, nch);
                for (unsigned long long c = c_lo; c < c_hi; c++) {
                    const unsigned long long base = c * kMmChunk;
                    const int cnt = (int)min((unsigned long long)kMmChunk, n - base);
                    float *dst = ring + (c % kMmSlots) * kMmChunk;
                    for (int i = t; i < cnt; i += nt) cp_async::ca4(dst + i, in + base + i);
                }
                cp_async::commit();
                cp_async::wait<0>();
                if (t == 0) sh_cnext = max(cnext, c_hi);
            }
        }
        __syncthreads();
        if (tid == 0) sh_lend = min(sh_cnext * kMmChunk, n);
    }
}

// ---- Decoder ------------------------------------------------------------------------------------------------------
__constant__ unsigned kChips[16] = {1618456172u, 1309113062u, 1826650030u, 1724778362u, 778887287u,  2061946375u,
                                    2007919840u, 125494990u,  529027475u,  838370585u,  320833617u,  422705285u,
                                    1368596360u, 85537272u,   139563807u,  2021988657u};
constexpr unsigned kMask = 0x7FFFFFFEu;
constexpr int kChipThreads = 256;
constexpr unsigned kMinFrameChips = 192;   // trigger, SFD, two header symbols, one byte: 6 x 32 chips

enum Mode : unsigned { kSearch = 0, kPreamble = 1, kSfd = 2, kHeader = 3, kDecode = 4 };

struct Frame {                         // == b2s_zigbee_frame
    unsigned long long index;
    unsigned len;
    int crc_ok;
    unsigned char bytes[128];
};
static_assert(sizeof(Frame) == sizeof(b2s_zigbee_frame), "ABI layout");

struct ZbState {
    unsigned long long pos0;           // stream index of the slice start
    unsigned long long n_fr;           // frames in the list
    unsigned sr;                       // the shift register after the last item (newest chip in bit 0)
    unsigned mode;
    unsigned next;                     // in a frame: where the next symbol is read, past the slice start
    int nib;                           // the first nibble of a byte (Option<u8>), -1 = None
    unsigned len, dlen;                // the header's length, bytes decoded so far
    unsigned char data[128];
};

__device__ __forceinline__ bool matching(unsigned sr, unsigned idx, unsigned thr) {
    return (unsigned)__popc((sr & kMask) ^ (kChips[idx] & kMask)) < thr;
}
// decode(): the first index of the smallest distance (min_by_key), if it is below the threshold; -1 otherwise
__device__ __forceinline__ int decode(unsigned sr, unsigned thr) {
    unsigned best = 33;
    int bi = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const unsigned d = __popc((sr & kMask) ^ (kChips[i] & kMask));
        if (d < best) { best = d; bi = i; }
    }
    return best < thr ? bi : -1;
}
// the shift register after item 32 w + k, from the chip words of items 32 w.. (cur) and 32 (w - 1).. (prev)
__device__ __forceinline__ unsigned shift_reg(unsigned cur, unsigned prev, unsigned k) {
    return (unsigned)(__brevll(((unsigned long long)cur << 32) | prev) >> (31 - k));
}

// chip words (bit k = item 32 w + k > 0) and Search triggers (matching(0) of the shift register at that item)
__global__ void __launch_bounds__(kChipThreads)
chips_kernel(const float *__restrict__ in, unsigned long long n, unsigned thr, const ZbState *__restrict__ st,
             unsigned *__restrict__ words, unsigned *__restrict__ trig) {
    const unsigned long long j = (unsigned long long)blockIdx.x * kChipThreads + threadIdx.x;
    const unsigned long long w = j >> 5;
    const unsigned lane = threadIdx.x & 31;
    if (w * 32 >= n) return;                           // whole warps only: the ballots need every lane
    const unsigned cur = __ballot_sync(~0u, j < n && in[j] > 0.0f);
    const unsigned prev = w ? __ballot_sync(~0u, in[j - 32] > 0.0f) : __brev(st->sr);
    const bool t = j < n && matching(shift_reg(cur, prev, lane), 0, thr);
    const unsigned tb = __ballot_sync(~0u, t);
    if (lane == 0) {
        words[w] = cur;
        trig[w] = tb;
    }
}

// Mac::calc_crc (mac.rs:62-80): CRC-16, reflected 0x1021, initial value 0
__device__ unsigned calc_crc(const unsigned char *d, unsigned len) {
    unsigned crc = 0;
    for (unsigned i = 0; i < len; i++)
        for (int k = 0; k < 8; k++) {
            const unsigned bit = ((d[i] >> k) & 1u) ^ (crc & 1u);
            crc >>= 1;
            if (bit) crc ^= 0x8408u;
        }
    return crc;
}

__global__ void __launch_bounds__(32)
walk_kernel(const unsigned *__restrict__ words, const unsigned *__restrict__ trig, unsigned long long n, unsigned thr,
            ZbState *__restrict__ st, Frame *__restrict__ frames) {
    __shared__ __align__(16) unsigned char data[128];
    const unsigned lane = threadIdx.x;
    const unsigned long long nw = (n + 31) / 32, pos0 = st->pos0, fr0 = st->n_fr;
    const unsigned carry = __brev(st->sr);
    for (unsigned i = lane; i < 128; i += 32) data[i] = st->data[i];
    unsigned mode = st->mode, len = st->len, dlen = st->dlen;
    int nib = st->nib;
    unsigned long long p = st->next, pos = 0, nfr = 0;
    auto sr_at = [&](unsigned long long q) {
        const unsigned long long w = q >> 5;
        return shift_reg(words[w], w ? words[w - 1] : carry, (unsigned)(q & 31));
    };
    const unsigned sr_end = sr_at(n - 1);
    __syncwarp();
    while (true) {
        if (mode == kSearch) {                         // the first trigger at or after pos
            unsigned long long t = n;
            for (unsigned long long w0 = pos >> 5; w0 < nw; w0 += 32) {
                const unsigned long long w = w0 + lane;
                unsigned m = w < nw ? trig[w] : 0u;
                if (w == (pos >> 5)) m &= ~0u << (pos & 31);
                const unsigned b = __ballot_sync(~0u, m != 0);
                if (b) {
                    const int l = __ffs(b) - 1;
                    const unsigned mm = __shfl_sync(~0u, m, l);
                    t = (w0 + l) * 32 + __ffs(mm) - 1;
                    break;
                }
            }
            if (t >= n) break;
            mode = kPreamble;                          // chip_count = 0: the next symbol is 32 chips on
            p = t + 32;
            continue;
        }
        if (p >= n) break;
        // the next 32 symbols of the frame, one per lane
        const unsigned long long q = p + 32ull * lane;
        unsigned info = 0;
        if (q < n) {
            const unsigned sr = sr_at(q);
            info = (unsigned)matching(sr, 0, thr) | (unsigned)matching(sr, 7, thr) << 1 |
                   (unsigned)matching(sr, 10, thr) << 2 | (unsigned)(decode(sr, thr) + 1) << 3;
        }
        const unsigned nv = (unsigned)min(32ull, (n - p + 31) / 32);
        unsigned k = 0;
        for (; k < nv; k++) {
            const unsigned v = __shfl_sync(~0u, info, k);
            const int dec = (int)(v >> 3) - 1;
            const unsigned long long qk = p + 32ull * k;
            if (mode == kPreamble) {
                if (v & 2u) mode = kSfd;
                else if (!(v & 1u)) mode = kSearch;
            } else if (mode == kSfd) {
                if (v & 4u) { mode = kHeader; nib = -1; }
                else mode = kSearch;
            } else if (dec < 0) {
                mode = kSearch;
            } else if (nib < 0) {
                nib = dec;
            } else if (mode == kHeader) {
                const unsigned l = ((unsigned)dec << 4) | (unsigned)nib;
                if (l < 128) { mode = kDecode; len = l; dlen = 0; nib = -1; }
                else mode = kSearch;
            } else {                                   // kDecode: a byte
                if (lane == 0 && dlen < 128) data[dlen] = (unsigned char)(((unsigned)dec << 4) | (unsigned)nib);
                if (dlen < 0xFFFFFFFFu) dlen++;
                nib = -1;
                if (dlen == len) {                     // post the frame; len 0 never gets here
                    __syncwarp();
                    Frame *f = frames + fr0 + nfr;
                    const unsigned *dw = reinterpret_cast<const unsigned *>(data);
                    unsigned word = dw[lane];
                    for (int b = 0; b < 4; b++)
                        if (lane * 4 + b >= len) word &= ~(0xFFu << (8 * b));
                    reinterpret_cast<unsigned *>(f->bytes)[lane] = word;
                    if (lane == 0) {
                        f->index = pos0 + qk;
                        f->len = len;
                        f->crc_ok = calc_crc(data, len) == 0 && len > 2;
                    }
                    __syncwarp();                      // every lane's read of data[] before lane 0 writes the next frame
                    nfr++;
                    mode = kSearch;
                }
            }
            if (mode == kSearch) { pos = qk + 1; break; }
        }
        if (mode != kSearch) p += 32ull * nv;
    }
    __syncwarp();
    for (unsigned i = lane; i < 128; i += 32) st->data[i] = data[i];
    if (lane == 0) {
        st->pos0 = pos0 + n;
        st->n_fr = fr0 + nfr;
        st->sr = sr_end;
        st->mode = mode;
        st->next = mode == kSearch ? 0u : (unsigned)(p - n);
        st->nib = nib;
        st->len = len;
        st->dlen = dlen;
    }
}

}  // namespace

struct b2s_mmclock {
    b2s_ctx *ctx = nullptr;
    MmParams prm{};
    MmState init{};
    Buf<MmState> st;
    Buf<MmState, Mem::Pinned> res;
};

struct b2s_zigbee {
    b2s_ctx *ctx = nullptr;
    unsigned thr = 6;
    Buf<ZbState> st;
    Buf<Frame> frames;
    Buf<unsigned> words, trig;
    size_t fr_bound = 0, fr_rd = 0;    // upper bound of the list's length, entries already drained
    ListCounts<1> counts;              // n_fr as the last exec left it
};

extern "C" {

// ---- ClockRecoveryMm --------------------------------------------------------------------------------------------
int32_t b2s_mmclock_create(b2s_ctx *ctx, float omega, float gain_omega, float mu, float gain_mu,
                           float omega_relative_limit, b2s_mmclock **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_mmclock_create: NULL argument");
    *out = nullptr;
    if (!std::isfinite(omega) || !std::isfinite(gain_omega) || !std::isfinite(mu) || !std::isfinite(gain_mu) ||
        !std::isfinite(omega_relative_limit))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_mmclock_create: parameters must be finite");
    const volatile float lim = omega * omega_relative_limit;     // f32 products and sums, as in new()
    if (!(lim >= 0.0f))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_mmclock_create: omega * omega_relative_limit = %g (f32::clamp needs >= 0)",
                        (double)lim);
    const volatile float s1 = omega + lim;
    const volatile float s2 = s1 + gain_mu;
    const float la_f = std::ceil((float)s2);
    const unsigned long long la = !(la_f > 0.0f) ? 0ull : la_f >= 18446744073709551616.0f ? ~0ull : (unsigned long long)la_f;
    if (la < 1)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_mmclock_create: look_ahead = ceil(omega + omega * omega_relative_limit + "
                        "gain_mu) = %llu (the loop reads i[ii + 1]: it must be >= 1)", la);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_mmclock> p(new b2s_mmclock());
    p->ctx = ctx;
    p->prm = MmParams{omega, (float)lim, gain_omega, gain_mu, la};
    p->init = MmState{omega, mu, 0.0f, 0, 0, 0};
    B2S_TRY(p->st.alloc(ctx, 1, "b2s_mmclock_create: state"));
    B2S_TRY(p->res.alloc(ctx, 1, "b2s_mmclock_create: result"));
    B2S_TRY(b2s_mmclock_reset(p.get()));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));          // `init` is copied from the plan itself
    *out = p.release();
    return B2S_OK;
}

void b2s_mmclock_destroy(b2s_mmclock *p) { PlanDeleter<b2s_mmclock>()(p); }

int32_t b2s_mmclock_reset(b2s_mmclock *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "mmclock is NULL");
    DeviceGuard g(p->ctx->device);
    B2S_CUDA(p->ctx, cudaMemcpyAsync(p->st.get(), &p->init, sizeof(MmState), cudaMemcpyHostToDevice, p->ctx->stream));
    return B2S_OK;
}

size_t b2s_mmclock_look_ahead(const b2s_mmclock *p) { return p ? (size_t)p->prm.look_ahead : 0; }

int32_t b2s_mmclock_exec(b2s_mmclock *p, const float *d_in, size_t n_in, float *d_out, size_t n_out_cap,
                         size_t *consumed, size_t *produced) {
    if (!p || !consumed || !produced) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_mmclock_exec: NULL argument");
    *consumed = *produced = 0;
    b2s_ctx *ctx = p->ctx;
    if (p->prm.look_ahead >= n_in || n_out_cap == 0) return B2S_OK;   // the loop does not run
    if (!d_in || !d_out) return b2s_fail(ctx, B2S_EINVAL, "b2s_mmclock_exec: NULL slice");
    if (!word_aligned(d_in) || !word_aligned(d_out))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_mmclock_exec: a slice is not 4-byte aligned");
    if (overlap(d_in, n_in * sizeof(float), d_out, n_out_cap * sizeof(float)))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_mmclock_exec: input and output overlap");
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_mmclock_exec");
    mm_kernel<<<1, kMmThreads, 0, ctx->stream>>>(d_in, n_in, d_out, n_out_cap, p->prm, p->st.get());
    B2S_CHECK_LAUNCH(ctx);
    B2S_CUDA(ctx, cudaMemcpyAsync(p->res.get(), p->st.get(), sizeof(MmState), cudaMemcpyDeviceToHost, ctx->stream));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const MmState r = *p->res.get();
    *consumed = (size_t)r.consumed;
    *produced = (size_t)r.produced;
    if (r.err)
        return b2s_fail(ctx, B2S_ESTATE, "b2s_mmclock_exec: step %zu would move ii past the slice (%zu items); the "
                        "block stopped before it", *produced, n_in);
    return B2S_OK;
}

// ---- Decoder ------------------------------------------------------------------------------------------------------
int32_t b2s_zigbee_create(b2s_ctx *ctx, uint32_t threshold, b2s_zigbee **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_zigbee_create: NULL argument");
    *out = nullptr;
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_zigbee> p(new b2s_zigbee());
    p->ctx = ctx;
    p->thr = threshold;
    B2S_TRY(p->st.alloc(ctx, 1, "b2s_zigbee_create: state"));
    B2S_TRY(p->counts.init(ctx, "b2s_zigbee_create: list count"));
    B2S_TRY(b2s_zigbee_reset(p.get()));
    *out = p.release();
    return B2S_OK;
}

void b2s_zigbee_destroy(b2s_zigbee *p) { PlanDeleter<b2s_zigbee>()(p); }

int32_t b2s_zigbee_reset(b2s_zigbee *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "zigbee is NULL");
    DeviceGuard g(p->ctx->device);
    B2S_TRY(b2s_memset(p->ctx, p->st.get(), 0, sizeof(ZbState)));
    B2S_TRY(b2s_memset(p->ctx, &p->st.get()->nib, 0xFF, sizeof(int)));   // None
    p->fr_bound = p->fr_rd = 0;
    p->counts.pending = false;
    return B2S_OK;
}

int32_t b2s_zigbee_exec(b2s_zigbee *p, const float *d_in, size_t n_in, size_t *consumed) {
    if (!p || !consumed) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_zigbee_exec: NULL argument");
    *consumed = 0;
    if (n_in == 0) return B2S_OK;
    b2s_ctx *ctx = p->ctx;
    if (!d_in) return b2s_fail(ctx, B2S_EINVAL, "b2s_zigbee_exec: NULL slice");
    if (!word_aligned(d_in)) return b2s_fail(ctx, B2S_EINVAL, "b2s_zigbee_exec: the slice is not 4-byte aligned");
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_zigbee_exec");
    const size_t nw = ceil_div(n_in, 32), bound_new = n_in / kMinFrameChips + 2;
    B2S_TRY(p->counts.refresh(ctx, p->frames.size() < p->fr_bound + bound_new, {&p->fr_bound}));
    B2S_TRY(list_grow(ctx, p->frames, p->fr_bound + bound_new, p->fr_bound, "b2s_zigbee_exec: frame list"));
    B2S_TRY(p->words.reserve(ctx, nw, "b2s_zigbee_exec: chip words"));
    B2S_TRY(p->trig.reserve(ctx, nw, "b2s_zigbee_exec: trigger bitmap"));
    ZbState *st = p->st.get();
    chips_kernel<<<(unsigned)ceil_div(nw * 32, kChipThreads), kChipThreads, 0, ctx->stream>>>(
        d_in, n_in, p->thr, st, p->words.get(), p->trig.get());
    B2S_CHECK_LAUNCH(ctx);
    walk_kernel<<<1, 32, 0, ctx->stream>>>(p->words.get(), p->trig.get(), n_in, p->thr, st, p->frames.get());
    B2S_CHECK_LAUNCH(ctx);
    B2S_TRY(p->counts.record(ctx, &st->n_fr));
    p->fr_bound += bound_new;
    *consumed = n_in;
    return B2S_OK;
}

int32_t b2s_zigbee_drain_frames(b2s_zigbee *p, b2s_zigbee_frame *host, size_t cap, size_t *n) {
    if (!p || !n || (cap && !host)) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_zigbee_drain_frames: NULL argument");
    return list_drain(p->ctx, p->frames, &p->st.get()->n_fr, p->counts, p->fr_rd, p->fr_bound, host, cap, n,
                      [](const Frame &) { return true; });
}

}  // extern "C"
