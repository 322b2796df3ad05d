// zigbee_tx.cu -- the ZigBee transmitter (examples/zigbee/src/mac.rs:135-252, modulator.rs:4-342 and iq_delay.rs:11-139,
// the chain of bin/tx.rs:37-56) as a device source (DESIGN §4.21).
//
// Framing stays on the host, inside push: a frame is at most 132 bytes, has no FEC, and its bytes are copied to the
// device anyway.  Push builds each frame (preamble, length, header with the sequence number, payload, FCS) and appends
// its bytes to a device byte ring; there is no encoder kernel.
//
// Exec (the hot path): the stream is cut into tiles of 1024-16384 samples, one CTA each.  Warp 0 finds the tile's first
// frame (tx_first_frame).  The CTA writes the pads as zero stores; for the part of a frame's body in its tile it puts
// the chip words of the bytes that part reads in shared memory, then writes each sample as a function of its offset k
// in the body: I is the modulator's sample k and Q its sample k - 2 (the two held Q values close the body).  A
// modulator sample is a DSSS chip of the byte's nibble (low first) times SHAPE[k % 4], formed in f32 as the reference
// forms it, so a negative chip at SHAPE 0.0 is -0.0.  Every sample is a function of its stream position and the frame
// records alone: execs never synchronise and any slicing gives the same stream.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "common.cuh"
#include "tx_common.cuh"

namespace {

constexpr unsigned kMaxPayload = B2S_ZIGBEE_MAX_PAYLOAD;   // MAX_FRAME_SIZE - 11 (mac.rs:155)
constexpr int kThreads = 256;
constexpr unsigned kTileMax = 16384;                      // stream samples per CTA: a large exec
constexpr unsigned kTileMin = 1024;                       // a small exec still spreads over every SM

// IEEE 802.15.4 O-QPSK chip sequences of symbols 0 and 8, chip c at bit 31 - c.  Symbol s (1-7, 9-15) is symbol 0 or
// 8 cyclically shifted right by 4 (s mod 8) chips; even chips go to I and odd chips to Q.  modulator.rs's DSSS table is
// these 16 rows as +-1 +- 1j (tests/golden/zigbee_tx_dsss.json).
constexpr uint32_t kChips0 = 0xD9C3522Eu;                  // 1101 1001 1100 0011 0101 0010 0010 1110
constexpr uint32_t kChips8 = 0x8C96077Bu;                  // 1000 1100 1001 0110 0000 0111 0111 1011

struct ZTxFrame {                      // device record of one queued frame
    unsigned long long start, byte_abs; // stream index of its first (front pad) sample; its first byte in the byte ring
    unsigned n_bytes, pad_;            // frame bytes: payload + 16
};

struct ExecParams {
    const uint8_t *bytes;
    unsigned long long byte_mask;
    const ZTxFrame *frames;
    unsigned long long frame_mask, f_lo;
    unsigned n_frames;                 // frames that [pos, pos + cnt) touches, from f_lo on
    unsigned long long pos, cnt;
    unsigned tile;                     // stream samples per CTA
    unsigned long long pad;            // IqDelay's PADDING, front and tail
    float2 *out;
};

// the chip word of a nibble: bit 31 - c is chip c
__device__ __forceinline__ uint32_t chip_word(unsigned nib) {
    const uint32_t base = nib < 8 ? kChips0 : kChips8;
    return __funnelshift_r(base, base, 4 * (nib & 7));
}

// modulator sample q of a frame, I (qbit 0) or Q (qbit 1): DSSS[nibble][chip] * SHAPE[q % 4] in f32, from the chip words
// w of the frame's nibbles from nibble 2 j0 on
__device__ __forceinline__ float chip_sample(const uint32_t *w, unsigned j0, unsigned q, unsigned qbit) {
    const unsigned c = 2 * ((q >> 2) & 15) + qbit;
    const float sign = (w[(q >> 6) - 2 * j0] >> (31 - c)) & 1 ? 1.0f : -1.0f;
    const unsigned p = q & 3;
    const float shape = p == 0 ? 0.0f : p == 2 ? 1.0f : 0.70710677f;   // SHAPE (modulator.rs:327)
    return __fmul_rn(sign, shape);
}

__global__ void __launch_bounds__(kThreads) zigbee_tx_exec_kernel(const ExecParams a) {
    __shared__ unsigned long long s_f;
    __shared__ uint32_t s_w[2 * (kTileMax / 128 + 3)];        // the chip words of the bytes a tile's body reads
    const unsigned long long t0 = a.pos + (unsigned long long)blockIdx.x * a.tile;
    const unsigned long long t1 = min(t0 + a.tile, a.pos + a.cnt);
    if (threadIdx.x < 32) {
        const unsigned long long f = tx_first_frame(a.frames, a.frame_mask, a.f_lo, a.n_frames, t0);
        if (threadIdx.x == 0) s_f = f;
    }
    __syncthreads();
    const auto zero = [](unsigned long long) { return make_float2(0.0f, 0.0f); };
    for (unsigned long long fi = s_f; fi < a.n_frames; ++fi) {
        const ZTxFrame fr = a.frames[(a.f_lo + fi) & a.frame_mask];
        if (fr.start >= t1) break;
        const unsigned nb = 128 * fr.n_bytes, body = nb + 2;       // modulator samples; IqDelay body with its Q tail
        const unsigned long long len = 2 * a.pad + body;
        const unsigned long long ra = max(t0, fr.start) - fr.start, rb = min(t1, fr.start + len) - fr.start;
        float2 *o = a.out + (fr.start - a.pos);
        store_range<kThreads>(o, ra, min(rb, a.pad), zero);
        store_range<kThreads>(o, max(ra, a.pad + body), rb, zero);
        const unsigned long long qa = max(ra, a.pad), qb = min(rb, a.pad + body);
        if (qa >= qb) continue;                                     // the same for every thread of the CTA
        // body samples [ka, kb) read the bytes j0..j1: I byte k / 128, Q byte (k - 2) / 128
        const unsigned ka = (unsigned)(qa - a.pad), kb = (unsigned)(qb - a.pad);
        const unsigned j0 = (ka < 2 ? 0 : ka - 2) >> 7, j1 = min((kb - 1) >> 7, fr.n_bytes - 1);
        __syncthreads();                                            // the previous frame's words are read
        for (unsigned t = threadIdx.x; t < 2 * (j1 - j0 + 1); t += kThreads) {
            const unsigned by = a.bytes[(fr.byte_abs + j0 + t / 2) & a.byte_mask];
            s_w[t] = chip_word((t & 1) ? by >> 4 : by & 15);         // low nibble first
        }
        __syncthreads();
        // IqDelay::work: o[k] = (m[k].re, m[k - 2].im), m[-2] = m[-1] = +0.0, then (0.0, m[nb - 2].im), (0.0, m[nb - 1].im)
        store_range<kThreads>(o + a.pad, ka, kb, [&](unsigned k) {
            const float i = k < nb ? chip_sample(s_w, j0, k, 0) : 0.0f;
            const float q = k >= 2 ? chip_sample(s_w, j0, k - 2, 1) : 0.0f;
            return make_float2(i, q);
        });
    }
}

// Mac::work's frame (mac.rs:203-221): 00 00 00 a7, n + 11, 41 88, seq, aa 1a ff ff 44 33, payload, calc_crc over
// bytes 5 .. 14 + n, little endian
void mac_frame(const uint8_t *payload, size_t n, unsigned seq, uint8_t *f) {
    const uint8_t hdr[14] = {0x00, 0x00, 0x00, 0xa7, (uint8_t)(n + 11), 0x41, 0x88, (uint8_t)seq,
                             0xaa, 0x1a, 0xff, 0xff, 0x44, 0x33};
    std::copy(hdr, hdr + 14, f);
    std::copy(payload, payload + n, f + 14);
    unsigned crc = 0;                                          // calc_crc (mac.rs:62-80)
    for (size_t i = 5; i < 14 + n; ++i)
        for (int k = 0; k < 8; ++k) {
            const unsigned bit = ((f[i] >> k) & 1u) ^ (crc & 1u);
            crc >>= 1;
            if (bit) crc ^= 0x8408u;                           // bits 15, 10 and 3
        }
    f[14 + n] = (uint8_t)(crc & 0xff);
    f[15 + n] = (uint8_t)(crc >> 8);
}

}  // namespace

struct b2s_zigbee_tx {
    b2s_ctx *ctx = nullptr;
    unsigned long long pad = 0;
    unsigned seq = 0;                  // Mac::sequence_number, a u8
    DevRing<uint8_t> bytes;
    DevRing<ZTxFrame> frames;
    TxQueue<b2s_zigbee_burst> q;

    unsigned long long frame_len(size_t n_bytes) const { return 2 * pad + 128ull * n_bytes + 2; }
};

extern "C" {

int32_t b2s_zigbee_tx_create(b2s_ctx *ctx, size_t pad, b2s_zigbee_tx **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_zigbee_tx_create: NULL argument");
    *out = nullptr;
    if (pad > 0xFFFFFFFFull) return b2s_fail(ctx, B2S_EINVAL, "b2s_zigbee_tx_create: pad %zu above 2^32 - 1", pad);
    PlanPtr<b2s_zigbee_tx> p(new b2s_zigbee_tx());
    p->ctx = ctx;
    p->pad = pad;
    *out = p.release();
    return B2S_OK;
}

void b2s_zigbee_tx_destroy(b2s_zigbee_tx *p) { PlanDeleter<b2s_zigbee_tx>()(p); }

int32_t b2s_zigbee_tx_reset(b2s_zigbee_tx *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "zigbee transmitter is NULL");
    p->q.reset();
    p->seq = 0;
    return B2S_OK;
}

int32_t b2s_zigbee_tx_push(b2s_zigbee_tx *p, const uint8_t *payloads, const size_t *lengths, size_t n_frames,
                           size_t *n_dropped) {
    if (!p || !n_dropped || (n_frames && !lengths))
        return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_zigbee_tx_push: NULL argument");
    b2s_ctx *ctx = p->ctx;
    *n_dropped = 0;
    size_t pay_bytes = 0;
    for (size_t i = 0; i < n_frames; ++i) pay_bytes += lengths[i];
    if (pay_bytes && !payloads) return b2s_fail(ctx, B2S_EINVAL, "b2s_zigbee_tx_push: NULL payloads");
    // Mac::tx drops an oversized payload on its own and keeps the rest (mac.rs:154-165); seq is taken per kept frame
    std::vector<uint8_t> fb;
    std::vector<ZTxFrame> rec;
    std::vector<TxHostFrame> hf;
    unsigned long long start = p->q.total, b = p->q.s_head;
    size_t off = 0, dropped = 0;
    const unsigned seq0 = p->seq;
    for (size_t i = 0; i < n_frames; off += lengths[i], ++i) {
        const size_t n = lengths[i];
        if (n > kMaxPayload) {
            ++dropped;
            continue;
        }
        const size_t k = fb.size();
        fb.resize(k + n + 16);
        mac_frame(payloads + off, n, p->seq, fb.data() + k);
        p->seq = (p->seq + 1) & 0xff;
        rec.push_back(ZTxFrame{start, b, (unsigned)(n + 16), 0});
        hf.push_back(TxHostFrame{start, p->frame_len(n + 16), b});
        start += hf.back().len;
        b += n + 16;
    }
    *n_dropped = dropped;
    if (rec.empty()) return B2S_OK;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_zigbee_tx_push");
    int32_t rc = p->frames.make_room(ctx, p->q.f_tail, p->q.f_head, rec.size(), "b2s_zigbee_tx_push: frame records");
    if (rc == B2S_OK) rc = p->bytes.make_room(ctx, p->q.s_tail, p->q.s_head, fb.size(), "b2s_zigbee_tx_push: frame bytes");
    if (rc == B2S_OK) rc = p->frames.put(ctx, p->q.f_head, rec.data(), rec.size());
    if (rc == B2S_OK) rc = p->bytes.put(ctx, p->q.s_head, fb.data(), fb.size());
    if (rc != B2S_OK) {
        p->seq = seq0;                                         // nothing was queued
        return rc;
    }
    p->q.append(hf, fb.size());
    return B2S_OK;
}

int32_t b2s_zigbee_tx_finish(b2s_zigbee_tx *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "zigbee transmitter is NULL");
    p->q.finishing = true;
    return B2S_OK;
}

int32_t b2s_zigbee_tx_pending(const b2s_zigbee_tx *p, uint64_t *samples) {
    if (!p || !samples) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_zigbee_tx_pending: NULL argument");
    *samples = p->q.total - p->q.pos;
    return B2S_OK;
}

int32_t b2s_zigbee_tx_exec(b2s_zigbee_tx *p, void *d_out, size_t n_out_cap, size_t *produced, int32_t *finished) {
    if (!p || !produced || !finished)
        return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_zigbee_tx_exec: NULL argument");
    b2s_ctx *ctx = p->ctx;
    *produced = 0;
    const unsigned long long cnt = std::min<unsigned long long>(n_out_cap, p->q.total - p->q.pos);
    if (cnt) {
        if (!d_out || ((uintptr_t)d_out & 7))
            return b2s_fail(ctx, B2S_EINVAL, "b2s_zigbee_tx_exec: output slice NULL or not 8-byte aligned");
        DeviceGuard g(ctx->device);
        NvtxRange nvtx("b2s_zigbee_tx_exec");
        const unsigned long long end = p->q.pos + cnt;
        ExecParams a;
        a.bytes = p->bytes.b.get();
        a.byte_mask = p->bytes.mask();
        a.frames = p->frames.b.get();
        a.frame_mask = p->frames.mask();
        a.f_lo = p->q.f_tail;
        a.n_frames = (unsigned)p->q.open(end);
        a.pos = p->q.pos;
        a.cnt = cnt;
        a.pad = p->pad;
        a.out = static_cast<float2 *>(d_out);
        // at least ~8 CTAs per SM where the exec is large enough; every tile size gives the same samples
        const size_t want = round_up(ceil_div(cnt, 8 * (size_t)std::max(ctx->sm_count, 1)), kTileMin);
        a.tile = (unsigned)std::min<size_t>(kTileMax, want);
        zigbee_tx_exec_kernel<<<(unsigned)ceil_div(cnt, a.tile), kThreads, 0, ctx->stream>>>(a);
        B2S_CHECK_LAUNCH(ctx);
        p->q.close(end);
        *produced = (size_t)cnt;
    }
    *finished = p->q.finished();
    return B2S_OK;
}

int32_t b2s_zigbee_tx_drain_bursts(b2s_zigbee_tx *p, b2s_zigbee_burst *host, size_t cap, size_t *n) {
    if (!p || !n || (cap && !host))
        return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_zigbee_tx_drain_bursts: NULL argument");
    *n = p->q.drain(host, cap);
    return B2S_OK;
}

}  // extern "C"
