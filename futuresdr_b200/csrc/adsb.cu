// adsb.cu -- the ADS-B receiver's PreambleDetector, Demodulator and Decoder::check_crc (examples/adsb/src/
// {preamble_detector,demodulator,decoder}.rs) as one fused device block.  Its tags never leave it as stream tags: they
// are the detection list, and the demodulated frames are the packet list (DESIGN §4.15).
//
// The detector scan (preamble_detector.rs:80-140) over positions pos < limit = L - 64:
//     if corr[pos] > thr * nf[pos]:  t0 = pos; idx = argmax_{j in t0..t0+31} corr[j] / nf[j] (strict >, first wins);
//                                   tag (idx, max) if the power check passes; pos = t0 + 31
//     else:                          pos += 1
// It is a finite-state walk: the only thing one position passes to the next is how far the last trigger's window
// still reaches, so a tile of T positions maps each of the 31 possible entry offsets to (exit offset, tags taken).
//   1. tile_kernel    one CTA per tile: ratio, trigger and power-check bitmaps in shared memory, then one lane per
//                     entry offset walks the trigger bitmap with __ffs -> the tile's transfer function.
//   2. group_kernel   one warp per group of kG tiles composes their functions (one lane per entry offset).
//   3. top_kernel     one warp walks the group functions from the carried scan offset: each group's entry and first
//                     tag ordinal, the scan end and the exec's tag count.
//   4. dist_kernel    one warp per group walks its tiles from the group's entry: each tile's entry and first ordinal.
//   5. emit_kernel    one warp per tile re-walks its bitmap from the true entry and writes its tags (argmax again)
//                     at their ordinals: in order, with no sorting and no atomics.
//   6. commit_kernel  one warp: which detections have their 480-sample window (the pending ones from earlier execs,
//                     then this exec's), the pending ones to carry, and the state for the next exec.
//   7. demod_kernel   one warp per demodulated detection: 112 PPM bits, the CRC-24 remainder and the 14 bytes.
// No step is serial in triggers or detections over the whole slice: a dense stream costs at most T/31 steps per
// tile.  Every exec is stream-ordered; only the two drain calls synchronise, and an exec whose worst case no longer fits
// a list's capacity (the list doubles; the bounds are tightened to the true counts once a copy of them has landed).
//
// Numerics: __fmul_rn / __fdiv_rn / __fadd_rn only and no FTZ, as in the reference's f32 (Rust neither contracts nor
// flushes).  NaN compares false, f32::min / f32::max are fminf / fmaxf (the non-NaN operand).
#include <algorithm>
#include <cstdint>

#include "lists.cuh"

namespace {

constexpr int kT = 4096;               // positions per tile
constexpr int kTW = kT / 32;           // bitmap words per tile
constexpr int kG = 128;                // tiles per group
constexpr int kE = 31;                 // entry offsets of a tile: 16 half-symbols x 2 samples - 1
constexpr int kTile = 256;             // threads of tile_kernel
constexpr int kChunk = 64;             // group functions top_kernel stages at a time
constexpr int kPend = 32;              // room for pending detections (at most 20 are ever pending, DESIGN §4.15)
constexpr unsigned kPreamble = 32;     // preamble_len_samples (demodulator.rs:64)
constexpr unsigned kPacket = 480;      // max_packet_len_samples (demodulator.rs:62)
constexpr unsigned kKeep = 544;        // an exec consumes L - 544: every tag below that has its window
constexpr size_t kMaxSlice = (size_t)1 << 30;   // positions looked at by one exec

struct Det {                           // == b2s_adsb_detection
    unsigned long long index;
    float value;
    unsigned pad;
};
struct Packet {                        // == b2s_adsb_packet
    unsigned long long index;
    float corr;
    int crc_passed;
    unsigned char bytes[14];
};
static_assert(sizeof(Det) == sizeof(b2s_adsb_detection) && sizeof(Packet) == sizeof(b2s_adsb_packet), "ABI layout");

struct State {
    unsigned long long pos0;           // stream index of the slice start
    unsigned long long n_det, n_pk;    // entries in the detection and packet lists
    unsigned off;                      // scan position past the slice start (< 600)
    unsigned np[2];                    // pending detections, by exec parity
    // written by top_kernel / commit_kernel for the rest of the exec
    unsigned scan_end, n_new, n_proc;
    unsigned long long det_base, pk_base, pos0_exec;
    Det pending[2][kPend];
};

// The scan from `pos` (relative to the tile) while pos < nt over the trigger bitmap `trig` (bits at nt and beyond are
// 0): on(t) for every trigger t taken, then pos = t + 31.  pos ends in [nt, nt + 30], or where it started if that is
// already >= nt.
template <class F> __device__ __forceinline__ void walk(const unsigned *trig, unsigned nt, unsigned &pos, F on) {
    while (pos < nt) {
        unsigned w = pos >> 5, m = trig[w] & (~0u << (pos & 31));
        while (!m && ++w < (unsigned)kTW) m = trig[w];
        const unsigned t = m ? w * 32 + __ffs(m) - 1 : nt;
        if (t >= nt) { pos = nt; break; }
        on(t);
        pos = t + kE;
    }
}
__device__ __forceinline__ bool bit(const unsigned *b, unsigned t) { return (b[t >> 5] >> (t & 31)) & 1u; }

// the 31-sample argmax of corr / nf from t0 (preamble_detector.rs:88-99); `ratio(j)` is corr[j] / nf[j]
template <class R> __device__ __forceinline__ unsigned argmax(R ratio, unsigned t0, float &mx) {
    mx = ratio(t0);
    unsigned idx = t0;
    for (unsigned j = t0 + 1; j < t0 + 32; j++) {
        const float r = ratio(j);
        if (r > mx) { mx = r; idx = j; }
    }
    return idx;
}

// the power check of preamble_detector.rs:102-125 on the 32 samples from idx
template <class S> __device__ __forceinline__ bool power_ok(S smp, unsigned idx) {
    float hmin = 0.f, hmax = 0.f, lmax = 0.f;
    int nh = 0, nl = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const float p = __fadd_rn(__fadd_rn(-0.0f, smp(idx + 2 * i)), smp(idx + 2 * i + 1));   // .sum::<f32>()
        if (i == 0 || i == 2 || i == 7 || i == 9) {
            hmin = nh ? fminf(hmin, p) : p;
            hmax = nh ? fmaxf(hmax, p) : p;
            nh++;
        } else {
            lmax = nl ? fmaxf(lmax, p) : p;
            nl++;
        }
    }
    return hmin > __fmul_rn(0.1f, hmax) && lmax < hmax;
}

__global__ void __launch_bounds__(kTile)
tile_kernel(const float *__restrict__ s, const float *__restrict__ nf, const float *__restrict__ corr,
            unsigned limit, float thr, const State *__restrict__ st, unsigned *__restrict__ bits,
            uint2 *__restrict__ tfun) {
    __shared__ float r[kT + 32];
    __shared__ float x[kT + 64];
    __shared__ unsigned trig[kTW], pass[kTW];
    const unsigned base = blockIdx.x * kT, nt = min((unsigned)kT, limit - base);
    const int tid = threadIdx.x, lane = tid & 31;
    // every index read below is < base + nt + 62 < limit + 64 = L
    for (int i = tid; i < kT + kTile; i += kTile) {   // whole warps every round: the ballot needs all lanes
        const unsigned p = base + i;
        bool t = false;
        if (i < (int)nt + 31 && i < kT + 32) {
            const float c = corr[p], n = nf[p];
            r[i] = __fdiv_rn(c, n);
            t = i < (int)nt && c > __fmul_rn(thr, n);
        }
        const unsigned b = __ballot_sync(~0u, t);
        if (lane == 0 && i < kT) trig[i >> 5] = b;
    }
    for (int i = tid; i < kT + 64; i += kTile)
        if (i < (int)nt + 63) x[i] = s[base + i];
    __syncthreads();
    for (int i = tid; i < kT; i += kTile) {
        bool ok = false;
        if (bit(trig, i)) {
            float mx;
            const unsigned idx = argmax([&](unsigned j) { return r[j]; }, (unsigned)i, mx);
            ok = power_ok([&](unsigned j) { return x[j]; }, idx);
        }
        const unsigned b = __ballot_sync(~0u, ok);
        if (lane == 0) pass[i >> 5] = b;
    }
    __syncthreads();
    if (tid < kTW) {
        bits[(size_t)blockIdx.x * 2 * kTW + tid] = trig[tid];
        bits[(size_t)blockIdx.x * 2 * kTW + kTW + tid] = pass[tid];
    }
    if (tid < 32) {
        // entry e of tile k > 0 is position base + e; tile 0 starts where the last exec's scan left off
        unsigned pos = blockIdx.x == 0 ? st->off : (unsigned)lane;
        unsigned cnt = 0;
        if (lane < kE) walk(trig, nt, pos, [&](unsigned t) { cnt += bit(pass, t); });
        tfun[(size_t)blockIdx.x * 32 + lane] = make_uint2(pos - nt, cnt);   // exit offset past the tile's end
    }
}

// groups of kG tile functions -> one function each (lane e: the walk entering the group's first tile at e)
__global__ void __launch_bounds__(32)
group_kernel(const uint2 *__restrict__ tfun, unsigned n_tiles, uint2 *__restrict__ gfun) {
    __shared__ uint2 f[kG * 32];
    const unsigned t0 = blockIdx.x * kG, nt = min((unsigned)kG, n_tiles - t0);
    for (unsigned i = threadIdx.x; i < nt * 32; i += 32) f[i] = tfun[(size_t)t0 * 32 + i];
    __syncwarp();
    unsigned e = threadIdx.x, cnt = 0;
    if (e < kE)
        for (unsigned t = 0; t < nt; t++) {
            const uint2 v = f[t * 32 + e];
            cnt += v.y;
            e = v.x;
        }
    gfun[(size_t)blockIdx.x * 32 + threadIdx.x] = make_uint2(e, cnt);
}

// the true walk over the groups; writes each group's (entry, first ordinal) and the exec's scan end and tag count
__global__ void __launch_bounds__(32)
top_kernel(const uint2 *__restrict__ gfun, unsigned n_groups, unsigned limit, uint2 *__restrict__ gent,
           State *__restrict__ st) {
    __shared__ uint2 f[kChunk * 32];
    unsigned e = 0, cnt = 0;           // group 0 holds tile 0, whose function ignores its entry
    for (unsigned g0 = 0; g0 < n_groups; g0 += kChunk) {
        const unsigned ng = min((unsigned)kChunk, n_groups - g0);
        __syncwarp();
        for (unsigned i = threadIdx.x; i < ng * 32; i += 32) f[i] = gfun[(size_t)g0 * 32 + i];
        __syncwarp();
        if (threadIdx.x == 0)
            for (unsigned g = 0; g < ng; g++) {
                gent[g0 + g] = make_uint2(e, cnt);
                const uint2 v = f[g * 32 + e];
                cnt += v.y;
                e = v.x;
            }
        e = __shfl_sync(~0u, e, 0);
        cnt = __shfl_sync(~0u, cnt, 0);
    }
    if (threadIdx.x == 0) {
        st->scan_end = n_groups ? limit + e : st->off;
        st->n_new = cnt;
    }
}

// each tile's (entry, first ordinal) from its group's
__global__ void __launch_bounds__(32)
dist_kernel(const uint2 *__restrict__ tfun, unsigned n_tiles, const uint2 *__restrict__ gent,
            uint2 *__restrict__ tent) {
    __shared__ uint2 f[kG * 32];
    const unsigned t0 = blockIdx.x * kG, nt = min((unsigned)kG, n_tiles - t0);
    for (unsigned i = threadIdx.x; i < nt * 32; i += 32) f[i] = tfun[(size_t)t0 * 32 + i];
    __syncwarp();
    if (threadIdx.x == 0) {
        uint2 g = gent[blockIdx.x];
        unsigned e = g.x, cnt = g.y;
        for (unsigned t = 0; t < nt; t++) {
            tent[t0 + t] = make_uint2(e, cnt);
            const uint2 v = f[t * 32 + (t0 + t == 0 ? 0 : e)];
            cnt += v.y;
            e = v.x;
        }
    }
}

// the tags of one tile, in order, at their ordinals
__global__ void __launch_bounds__(32)
emit_kernel(const float *__restrict__ nf, const float *__restrict__ corr, unsigned limit,
            const unsigned *__restrict__ bits, const uint2 *__restrict__ tent, const State *__restrict__ st,
            Det *__restrict__ dets) {
    __shared__ unsigned trig[kTW], pass[kTW];
    __shared__ unsigned list[kT / kE + 2];
    __shared__ unsigned n_list;
    const unsigned base = blockIdx.x * kT, nt = min((unsigned)kT, limit - base);
    for (unsigned i = threadIdx.x; i < kTW; i += 32) {
        trig[i] = bits[(size_t)blockIdx.x * 2 * kTW + i];
        pass[i] = bits[(size_t)blockIdx.x * 2 * kTW + kTW + i];
    }
    __syncwarp();
    const uint2 te = tent[blockIdx.x];
    if (threadIdx.x == 0) {
        unsigned pos = blockIdx.x == 0 ? st->off : te.x, n = 0;
        walk(trig, nt, pos, [&](unsigned t) { if (bit(pass, t)) list[n++] = t; });
        n_list = n;
    }
    __syncwarp();
    const unsigned n = n_list;
    const unsigned long long d0 = st->n_det + te.y, pos0 = st->pos0;
    for (unsigned j = threadIdx.x; j < n; j += 32) {
        float mx;
        const unsigned idx = argmax([&](unsigned k) { return __fdiv_rn(corr[base + k], nf[base + k]); }, list[j], mx);
        dets[d0 + j] = Det{pos0 + base + idx, mx, 0u};
    }
}

// Which detections have their window: the pending ones carried from earlier execs, then this exec's, in index order.
// Non-final: g < pos0 + c (then g + 480 < c + 480 < L - 64 <= scan end).  Final: g + 480 < D, D = the scan end.
__global__ void __launch_bounds__(32)
commit_kernel(State *__restrict__ st, const Det *__restrict__ dets, int par, int final, unsigned long long c) {
    const unsigned np = st->np[par], total = np + st->n_new;
    const unsigned long long pos0 = st->pos0, n_det = st->n_det, d_end = pos0 + st->scan_end;
    auto get = [&](unsigned i) { return i < np ? st->pending[par][i] : dets[n_det + i - np]; };
    auto ready = [&](unsigned long long g) { return final ? g + kPacket < d_end : g < pos0 + c; };
    unsigned lo = 0;
    if (threadIdx.x == 0) {                    // the list is sorted by index: the ready ones are a prefix
        unsigned hi = total;
        while (lo < hi) {
            const unsigned mid = (lo + hi) / 2;
            if (ready(get(mid).index)) lo = mid + 1;
            else hi = mid;
        }
    }
    const unsigned n_proc = __shfl_sync(~0u, lo, 0);
    const unsigned keep = final ? 0u : min(total - n_proc, (unsigned)kPend);
    if (threadIdx.x < keep) st->pending[par ^ 1][threadIdx.x] = get(n_proc + threadIdx.x);
    __syncwarp();
    if (threadIdx.x == 0) {
        st->det_base = n_det;
        st->pk_base = st->n_pk;
        st->pos0_exec = pos0;
        st->n_proc = n_proc;
        st->np[par ^ 1] = keep;
        st->n_det = n_det + st->n_new;
        st->n_pk += n_proc;
        if (!final) {
            st->off = st->scan_end - (unsigned)c;
            st->pos0 = pos0 + c;
        }
    }
}

// Demodulator::work (demodulator.rs:66-92) and Decoder::check_crc (decoder.rs:57-73) for detection w of the ready
// prefix: bit s compares fold(0.0, acc + x * tap) over the 4 samples from g + 32 + 4 s with the ZERO and ONE taps.
__global__ void __launch_bounds__(128)
demod_kernel(const float *__restrict__ s, const State *__restrict__ st, const Det *__restrict__ dets, int par,
             Packet *__restrict__ pk) {
    const unsigned w = blockIdx.x * 4 + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (w >= st->n_proc) return;
    const unsigned np = st->np[par];
    const Det d = w < np ? st->pending[par][w] : dets[st->det_base + w - np];
    const float *x = s + (d.index - st->pos0_exec) + kPreamble;
    unsigned m[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const unsigned sym = q * 32 + lane;
        bool one = false;
        if (sym < 112) {
            const float *y = x + 4 * sym;
            float c0 = 0.0f, c1 = 0.0f;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const float v = y[i];
                c0 = __fadd_rn(c0, __fmul_rn(v, i < 2 ? -1.0f : 1.0f));    // SYMBOL_ZERO_TAPS
                c1 = __fadd_rn(c1, __fmul_rn(v, i < 2 ? 1.0f : -1.0f));    // SYMBOL_ONE_TAPS
            }
            one = !(c0 > c1);
        }
        m[q] = __ballot_sync(~0u, one);
    }
    if (lane == 0) {
        Packet p;
        unsigned rem = 0;                      // long division by the 25-bit generator 0x1FFF409
        for (int b = 0; b < 112; b++) {
            rem = (rem << 1) | ((m[b >> 5] >> (b & 31)) & 1u);
            if (rem & (1u << 24)) rem ^= 0x1FFF409u;
        }
        for (int k = 0; k < 14; k++) {         // bin_to_u64 over 8 bits, MSB first
            unsigned v = 0;
            for (int b = 8 * k; b < 8 * k + 8; b++) v = (v << 1) | ((m[b >> 5] >> (b & 31)) & 1u);
            p.bytes[k] = (unsigned char)v;
        }
        p.index = d.index;
        p.corr = d.value;
        p.crc_passed = rem == 0;
        pk[st->pk_base + w] = p;
    }
}

}  // namespace

struct b2s_adsb {
    b2s_ctx *ctx = nullptr;
    float thr = 10.0f;
    bool forward_failed_crc = false;
    Buf<State> st;
    Buf<Det> dets;
    Buf<Packet> pks;
    Buf<unsigned> bits;                // per tile: trigger bitmap, then power-check bitmap
    Buf<uint2> tfun, gfun, gent, tent; // transfer functions of tiles / groups, entries of groups / tiles
    size_t det_bound = 0, pk_bound = 0;   // upper bounds of the device lists' lengths
    size_t det_rd = 0, pk_rd = 0;         // entries already drained
    ListCounts<2> counts;                 // (n_det, n_pk) as the last exec left them
    int par = 0;
    bool done = false;
};

namespace {

int32_t clear(b2s_adsb *p) {
    B2S_TRY(b2s_memset(p->ctx, p->st.get(), 0, sizeof(State)));
    p->det_bound = p->pk_bound = p->det_rd = p->pk_rd = 0;
    p->counts.pending = false;
    p->par = 0;
    p->done = false;
    return B2S_OK;
}

}  // namespace

extern "C" {

int32_t b2s_adsb_create(b2s_ctx *ctx, float threshold, int32_t forward_failed_crc, b2s_adsb **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_adsb_create: NULL argument");
    *out = nullptr;
    if (!(threshold >= 0.0f) || threshold == INFINITY)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_adsb_create: threshold %g (a finite value >= 0)", (double)threshold);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_adsb> p(new b2s_adsb());
    p->ctx = ctx;
    p->thr = threshold;
    p->forward_failed_crc = forward_failed_crc != 0;
    B2S_TRY(p->st.alloc(ctx, 1, "b2s_adsb_create: state"));
    B2S_TRY(p->counts.init(ctx, "b2s_adsb_create: list counts"));
    B2S_TRY(clear(p.get()));
    *out = p.release();
    return B2S_OK;
}

void b2s_adsb_destroy(b2s_adsb *p) { PlanDeleter<b2s_adsb>()(p); }

int32_t b2s_adsb_reset(b2s_adsb *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "adsb is NULL");
    DeviceGuard g(p->ctx->device);
    return clear(p);
}

int32_t b2s_adsb_exec(b2s_adsb *p, const float *d_samples, size_t n_samples, const float *d_nf, size_t n_nf,
                      const float *d_corr, size_t n_corr, int32_t finished, size_t *consumed, int32_t *done) {
    if (!p || !consumed || !done) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_adsb_exec: NULL argument");
    *consumed = 0;
    *done = p->done;
    if (p->done) return B2S_OK;
    b2s_ctx *ctx = p->ctx;
    size_t L = std::min({n_samples, n_nf, n_corr});
    const bool final = finished && L <= kMaxSlice;
    L = std::min(L, kMaxSlice);
    if (L && (!d_samples || !d_nf || !d_corr)) return b2s_fail(ctx, B2S_EINVAL, "b2s_adsb_exec: NULL slice");
    if (L && (!word_aligned(d_samples) || !word_aligned(d_nf) || !word_aligned(d_corr)))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_adsb_exec: a slice is not 4-byte aligned");
    const size_t limit = sat_sub(L, 64), c = final ? L : sat_sub(L, kKeep);
    if (!final && limit == 0) return B2S_OK;                 // nothing to scan and nothing ready
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_adsb_exec");
    const unsigned n_tiles = (unsigned)ceil_div(limit, kT), n_groups = (unsigned)ceil_div(n_tiles, kG);
    const size_t bound_new = limit / kE + 1;                 // triggers are >= 31 positions apart
    // the counts behind the last exec tighten the bounds once they have landed; an exec that would have to grow a list
    // waits for them first (growing synchronises anyway), so the capacity follows the true lengths
    const bool tight = p->dets.size() >= p->det_bound + bound_new && p->pks.size() >= p->pk_bound + kPend + bound_new;
    B2S_TRY(p->counts.refresh(ctx, !tight, {&p->det_bound, &p->pk_bound}));
    B2S_TRY(list_grow(ctx, p->dets, p->det_bound + bound_new, p->det_bound, "b2s_adsb_exec: detection list"));
    B2S_TRY(list_grow(ctx, p->pks, p->pk_bound + kPend + bound_new, p->pk_bound, "b2s_adsb_exec: packet list"));
    if (n_tiles) {
        B2S_TRY(p->bits.reserve(ctx, (size_t)n_tiles * 2 * kTW, "b2s_adsb_exec: bitmaps"));
        B2S_TRY(p->tfun.reserve(ctx, (size_t)n_tiles * 32, "b2s_adsb_exec: tile functions"));
        B2S_TRY(p->tent.reserve(ctx, n_tiles, "b2s_adsb_exec: tile entries"));
        B2S_TRY(p->gfun.reserve(ctx, (size_t)n_groups * 32, "b2s_adsb_exec: group functions"));
        B2S_TRY(p->gent.reserve(ctx, n_groups, "b2s_adsb_exec: group entries"));
    }
    State *st = p->st.get();
    cudaStream_t s = ctx->stream;
    if (n_tiles) {
        tile_kernel<<<n_tiles, kTile, 0, s>>>(d_samples, d_nf, d_corr, (unsigned)limit, p->thr, st, p->bits.get(),
                                               p->tfun.get());
        B2S_CHECK_LAUNCH(ctx);
        group_kernel<<<n_groups, 32, 0, s>>>(p->tfun.get(), n_tiles, p->gfun.get());
        B2S_CHECK_LAUNCH(ctx);
    }
    top_kernel<<<1, 32, 0, s>>>(p->gfun.get(), n_groups, (unsigned)limit, p->gent.get(), st);
    B2S_CHECK_LAUNCH(ctx);
    if (n_tiles) {
        dist_kernel<<<n_groups, 32, 0, s>>>(p->tfun.get(), n_tiles, p->gent.get(), p->tent.get());
        B2S_CHECK_LAUNCH(ctx);
        emit_kernel<<<n_tiles, 32, 0, s>>>(d_nf, d_corr, (unsigned)limit, p->bits.get(), p->tent.get(), st,
                                            p->dets.get());
        B2S_CHECK_LAUNCH(ctx);
    }
    commit_kernel<<<1, 32, 0, s>>>(st, p->dets.get(), p->par, final, (unsigned long long)c);
    B2S_CHECK_LAUNCH(ctx);
    const size_t warps = kPend + bound_new;
    demod_kernel<<<(unsigned)ceil_div(warps, 4), 128, 0, s>>>(d_samples, st, p->dets.get(), p->par, p->pks.get());
    B2S_CHECK_LAUNCH(ctx);
    static_assert(offsetof(State, n_pk) == offsetof(State, n_det) + sizeof(unsigned long long), "counts copy");
    B2S_TRY(p->counts.record(ctx, &st->n_det));
    p->det_bound += bound_new;
    p->pk_bound += kPend + bound_new;
    p->par ^= 1;
    p->done = final;
    *consumed = c;
    *done = final;
    return B2S_OK;
}

int32_t b2s_adsb_drain_packets(b2s_adsb *p, b2s_adsb_packet *host, size_t cap, size_t *n) {
    if (!p || !n || (cap && !host)) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_adsb_drain_packets: NULL argument");
    const bool all = p->forward_failed_crc;
    return list_drain(p->ctx, p->pks, &p->st.get()->n_pk, p->counts, p->pk_rd, p->pk_bound, host, cap, n,
                 [all](const Packet &e) { return all || e.crc_passed; });
}

int32_t b2s_adsb_drain_detections(b2s_adsb *p, b2s_adsb_detection *host, size_t cap, size_t *n) {
    if (!p || !n || (cap && !host)) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_adsb_drain_detections: NULL argument");
    return list_drain(p->ctx, p->dets, &p->st.get()->n_det, p->counts, p->det_rd, p->det_bound, host, cap, n,
                 [](const Det &) { return true; });
}

}  // extern "C"
