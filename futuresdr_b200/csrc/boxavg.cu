// boxavg.cu -- the WLAN and M17 receivers' MovingAverage (examples/wlan/src/moving_average.rs:44-107,
// examples/m17/src/moving_average.rs:20-81): a running sum over `len` items, restarted at every work() call.
// Not the library's MovingAvg (mavg.cu), which is an exponential average per bin.
//
// One work() call with pad == 0 produces m = min(4000, n_in + 1 - len, n_out) outputs from a strict-order f32 chain:
//     sum = fold(+, init, x[0 .. len-1]);  for i in 0..m { sum += x[i+len-1]; out[i] = sum [/ div]; sum -= x[i]; }
// init is -0.0 for f32 (the std `Sum<&f32>` of Rust 1.83 and later, which the 2024-edition reference needs) and
// Complex32::zero() = (+0, +0) for Complex32 (num_complex folds from zero).  The rounding of every output depends on
// where the calls fall, so nothing here reassociates: each call is one sequential chain, a "segment".
//
// One exec emulates the calls the reference makes back to back on the remaining slices (the host does the
// bookkeeping, see b2s_boxavg_exec): the remaining pad is a memset, then segments of 4000 outputs, of which only the
// last may be shorter.  Segment s reads x[4000 s ..) and writes out[pad + 4000 s ..).  All segments are independent,
// so the parallelism is across segments and each chain runs on one lane (Complex32: one lane per component).
//
// Layout.  One warp per CTA owns 32 / W consecutive segments (W = 32-bit words per item).  Each segment's stream
// y[j] = x[4000 s + j], j < len - 1 + m, is walked in tiles of K items.  A tile of all the CTA's segments is copied
// into shared memory with 4-byte cp.async, consecutive lanes on consecutive words of one segment's row (coalesced at
// any 4-byte alignment), kStages tiles ahead of the chain.  The row pitch P = (K + 1) W words puts the lanes of a
// transposed step -- lane r W + c reads word j W + c of row r -- on 32 distinct banks.  Output words are written to a
// tile of the same shape and leave through shared memory, again as coalesced rows.
//
// The trailing stream x[i] is the leading stream delayed by len - 1 steps.  Short windows (len - 1 <= kRingItems)
// keep the last ceil((len-1)/K) lead tiles resident and read the trailing item from them: every input item crosses HBM
// once.  Longer windows (M17's 4800) load the trailing stream as a second tile stream, and the lead stream of a
// segment also covers its len - 1 item prefix: about 2 + (len-1)/4000 input reads per item (DESIGN §4.14).
//
// Numerics: __fadd_rn / __fsub_rn / __fdiv_rn only, no FTZ (the library is built without --use_fast_math), so signed
// zeros, denormals, infinities and NaN follow IEEE exactly; an inf entering the sum becomes NaN when it leaves it,
// and the NaN lasts until the end of that segment, as in the reference.
#include <algorithm>
#include <cstdint>

#include "common.cuh"

namespace {

constexpr size_t kMaxIter = 4000;     // MAX_ITER (moving_average.rs:3)
constexpr int kK = 32;                // items per tile row
constexpr int kStages = 4;            // tiles in flight ahead of the chain
constexpr int kRingItems = 4 * kK;    // len - 1 up to which the trailing stream comes from the resident lead tiles

template <int W> struct Geo {
    static constexpr int rows = 32 / W;           // segments per CTA
    static constexpr int KW = kK * W;             // words of one row of a tile
    static constexpr int P = KW + W;              // row pitch: lane r W + c lands on bank (r W + c + const) mod 32
    static constexpr int tile = rows * P;         // floats per tile (1056 for both item widths)
};

// n_seg segments; all hold 4000 outputs but the last, which holds m_last.  c0 = len - 1.  ring: lead tiles resident
// (RING) or in flight (otherwise).  Shared memory: `ring` lead tiles, kStages trailing tiles (not RING), 1 output tile.
template <int W, bool RING, bool DIV>
__global__ void __launch_bounds__(32)
boxavg_kernel(const float *__restrict__ in, float *__restrict__ out, unsigned long long n_seg, unsigned m_last,
              unsigned c0, float div, int ring) {
    using G = Geo<W>;
    extern __shared__ float sm[];
    float *lead = sm;
    float *trail = sm + ring * G::tile;
    float *outt = sm + (ring + (RING ? 0 : kStages)) * G::tile;

    const int lane = threadIdx.x, r = lane / W, c = lane % W;
    const unsigned long long seg0 = (unsigned long long)blockIdx.x * G::rows;
    const int rows_here = (int)min((unsigned long long)G::rows, n_seg - seg0);
    const int last_row = (int)min((unsigned long long)G::rows, n_seg - 1 - seg0);   // == rows if not in this CTA
    const unsigned mmax = last_row == 0 ? m_last : (unsigned)kMaxIter;             // row 0 is the longest row
    const unsigned J = c0 + mmax;                                                  // steps of the longest chain
    const unsigned T = (J + kK - 1) / kK;                                          // tiles
    const float *in0 = in + seg0 * kMaxIter * W;
    float *out0 = out + seg0 * kMaxIter * W;

    // Tile t of every row: lead items [tK, tK + K), and (not RING) trailing items [tK - c0, tK - c0 + K).  Lane word
    // w of row rr is word w of that row's K W-word window; k enumerates (rr, w) so that w = lane + 32 (k mod W).
    auto issue = [&](unsigned t) {
        if (t < T) {
            float *L = lead + (t % ring) * G::tile;
            float *Tr = trail + (t % kStages) * G::tile;
#pragma unroll
            for (int k = 0; k < 32; k++) {
                const int rr = k / W, w = lane + 32 * (k % W);
                if (rr < rows_here) {
                    const unsigned m = rr == last_row ? m_last : (unsigned)kMaxIter;
                    const unsigned it = t * kK + w / W;
                    const float *src = in0 + (size_t)rr * kMaxIter * W + (size_t)t * G::KW + w;
                    if (it < c0 + m) cp_async::ca4(L + rr * G::P + w, src);
                    if (!RING && it >= c0 && it - c0 < m) cp_async::ca4(Tr + rr * G::P + w, src - (size_t)c0 * W);
                }
            }
        }
        cp_async::commit();                    // one group per tile, empty ones included, so wait_group counts tiles
    };

#pragma unroll
    for (int p = 0; p < kStages - 1; p++) issue(p);

    const unsigned q = c0 / kK, rem = c0 % kK;
    float s = W == 1 ? -0.0f : 0.0f;
    for (unsigned t = 0; t < T; t++) {
        issue(t + kStages - 1);
        cp_async::wait<kStages - 1>();         // tile t has landed (this lane's copies) ...
        __syncwarp();                          // ... and every lane's
        const float *Lr = lead + (t % ring) * G::tile + r * G::P + c;
        const float *pA, *pB;                  // trailing item of step jj: pA[jj W] for jj < rem, else pB[jj W]
        if (RING) {                            // item tK + jj - c0 lies in tile t - q (jj >= rem) or t - q - 1
            const int sb = (int)(((long long)t - q) % ring + ring) % ring;
            const int sa = (sb + ring - 1) % ring;
            pB = lead + sb * G::tile + r * G::P + c - (int)rem * W;
            pA = lead + sa * G::tile + r * G::P + c + (kK - (int)rem) * W;
        } else {
            pB = trail + (t % kStages) * G::tile + r * G::P + c;
            pA = pB;
        }
        float *Or = outt + r * G::P + c;
        const unsigned j0 = t * kK;
        if (j0 >= c0 && j0 + kK <= J) {        // the steady state: a whole tile of outputs
#pragma unroll
            for (int jj = 0; jj < kK; jj++) {
                s = __fadd_rn(s, Lr[jj * W]);
                Or[jj * W] = DIV ? __fdiv_rn(s, div) : s;
                s = __fsub_rn(s, (RING && jj < (int)rem ? pA : pB)[jj * W]);
            }
        } else {                               // prefix, the tile where outputs start, or the last tile
            for (int jj = 0; jj < kK && j0 + jj < J; jj++) {
                s = __fadd_rn(s, Lr[jj * W]);
                if (j0 + jj >= c0) {
                    Or[jj * W] = DIV ? __fdiv_rn(s, div) : s;
                    s = __fsub_rn(s, (RING && jj < (int)rem ? pA : pB)[jj * W]);
                }
            }
        }
        __syncwarp();
        if (j0 + kK > c0) {                    // rows of outputs i = tK + jj - c0, 0 <= i < m
#pragma unroll
            for (int k = 0; k < 32; k++) {
                const int rr = k / W, w = lane + 32 * (k % W);
                if (rr < rows_here) {
                    const unsigned m = rr == last_row ? m_last : (unsigned)kMaxIter;
                    const long long i = (long long)j0 + w / W - c0;
                    if (i >= 0 && i < (long long)m)
                        out0[(size_t)rr * kMaxIter * W + (size_t)i * W + (w % W)] = outt[rr * G::P + w];
                }
            }
        }
        __syncwarp();                          // the output tile and tile t's slots are free again
    }
    cp_async::wait<0>();
}

template <int W, bool RING, bool DIV>
int32_t launch(b2s_ctx *ctx, const float *in, float *out, size_t n_seg, unsigned m_last, unsigned c0, float div) {
    using G = Geo<W>;
    const int ring = RING ? kStages + (int)ceil_div(c0, kK) : kStages;
    const size_t smem = (size_t)(ring + (RING ? 0 : kStages) + 1) * G::tile * sizeof(float);
    constexpr auto kernel = boxavg_kernel<W, RING, DIV>;
    B2S_TRY(smem_optin<kernel>(ctx, smem));
    const size_t grid = ceil_div(n_seg, G::rows);
    if (grid > 0x7FFFFFFFu) return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_boxavg_exec: %zu segments in one exec", n_seg);
    kernel<<<(unsigned)grid, 32, smem, ctx->stream>>>(in, out, n_seg, m_last, c0, div, ring);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

}  // namespace

struct b2s_boxavg {
    b2s_ctx *ctx = nullptr;
    bool cplx = false;
    size_t len = 1;
    bool has_div = false;
    float div = 1.0f;
    size_t pad = 0;                    // zeros still to emit (moving_average.rs:38, starts at len - 1)
};

extern "C" {

int32_t b2s_boxavg_create(b2s_ctx *ctx, int32_t complex_items, size_t len, int32_t has_divisor, float divisor,
                          b2s_boxavg **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_boxavg_create: NULL argument");
    *out = nullptr;
    if (len == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_boxavg_create: len == 0 (moving_average.rs asserts len > 0)");
    if (len > ((size_t)1 << 31))
        return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_boxavg_create: len %zu (at most 2^31)", len);
    if (complex_items && has_divisor)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_boxavg_create: a divisor needs f32 items (no Complex32 block divides)");
    PlanPtr<b2s_boxavg> p(new b2s_boxavg());
    p->ctx = ctx;
    p->cplx = complex_items != 0;
    p->len = len;
    p->has_div = has_divisor != 0;
    p->div = divisor;
    p->pad = len - 1;
    *out = p.release();
    return B2S_OK;
}

void b2s_boxavg_destroy(b2s_boxavg *p) { PlanDeleter<b2s_boxavg>()(p); }

int32_t b2s_boxavg_reset(b2s_boxavg *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "boxavg is NULL");
    p->pad = p->len - 1;
    return B2S_OK;
}

int32_t b2s_boxavg_exec(b2s_boxavg *p, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                        size_t max_calls, size_t *consumed, size_t *produced, size_t *calls, int32_t *call_again,
                        int32_t *done) {
    if (!p || !consumed || !produced || !calls || !call_again || !done)
        return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_boxavg_exec: NULL argument");
    *consumed = *produced = *calls = 0;
    *call_again = *done = 0;
    b2s_ctx *ctx = p->ctx;
    // the work() calls, back to back on what is left of the slices (moving_average.rs:76-104)
    size_t pad = p->pad, c = 0, prod = 0, n_calls = 0, pad_items = 0, n_seg = 0, m_last = 0;
    bool again = false, fin = false;
    while (max_calls == 0 || n_calls < max_calls) {
        n_calls++;
        const size_t rem_out = n_out_cap - prod;
        if (pad > 0) {                                         // :76-85
            const size_t m = std::min(pad, rem_out);
            pad -= m;
            pad_items += m;
            prod += m;
            again = m < rem_out;
            fin = false;
            if (m == 0) break;
        } else {                                               // :86-103
            const size_t avail = sat_sub(n_in - c + 1, p->len);
            const size_t m = std::min(std::min(kMaxIter, avail), rem_out);
            again = false;
            fin = m == avail;
            if (m == 0) break;
            n_seg++;
            m_last = m;
            c += m;
            prod += m;
        }
    }
    const size_t isz = p->cplx ? 8 : 4;
    if (pad_items || n_seg) {
        if (!d_out || (n_seg && !d_in)) return b2s_fail(ctx, B2S_EINVAL, "b2s_boxavg_exec: NULL slice");
        if (!word_aligned(d_out) || (n_seg && !word_aligned(d_in)))
            return b2s_fail(ctx, B2S_EINVAL, "b2s_boxavg_exec: a slice is not 4-byte aligned");
    }
    if (n_seg && overlap(d_in, (c + p->len - 1) * isz, d_out, prod * isz))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_boxavg_exec: the output overlaps the input");
    if (pad_items || n_seg) {
        DeviceGuard g(ctx->device);
        NvtxRange nvtx("b2s_boxavg_exec");
        if (pad_items) B2S_TRY(b2s_memset(ctx, d_out, 0, pad_items * isz));     // out[0..m].fill(zero)
        if (n_seg) {
            const float *in = (const float *)d_in;
            float *o = (float *)((char *)d_out + pad_items * isz);
            const unsigned c0 = (unsigned)(p->len - 1), ml = (unsigned)m_last;
            const bool ring = c0 <= (unsigned)kRingItems;
            int32_t rc;
            if (p->cplx) rc = ring ? launch<2, true, false>(ctx, in, o, n_seg, ml, c0, 0.f)
                                   : launch<2, false, false>(ctx, in, o, n_seg, ml, c0, 0.f);
            else if (p->has_div) rc = ring ? launch<1, true, true>(ctx, in, o, n_seg, ml, c0, p->div)
                                           : launch<1, false, true>(ctx, in, o, n_seg, ml, c0, p->div);
            else rc = ring ? launch<1, true, false>(ctx, in, o, n_seg, ml, c0, 0.f)
                           : launch<1, false, false>(ctx, in, o, n_seg, ml, c0, 0.f);
            B2S_TRY(rc);
        }
    }
    p->pad = pad;
    *consumed = c;
    *produced = prod;
    *calls = n_calls;
    *call_again = again;
    *done = fin;
    return B2S_OK;
}

}  // extern "C"
