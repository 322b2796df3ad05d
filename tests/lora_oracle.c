/* CPU oracle of the LoRa transmitter (TEST INFRASTRUCTURE ONLY): examples/lora/src/encoder.rs:33-284 (Encoder::encode),
 * utils.rs:917-963 (build_upchirp_phase_coherent, samples_from_phase_diff), modulator.rs:46-152 (Modulator::modulate)
 * and utils.rs:988-1020 (sample_count), one reference call at a time, in the reference's types and operation order.
 * cos / sin are libm's cosf / sinf, which Rust's f32::cos / f32::sin call.  The reference's LoRa code has no tests, so
 * this parity is unpinned: it is cross-checked against the Python transcription in tests/lora_oracle.py. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

static uint8_t whitening_seq(size_t i) { /* WHITENING_SEQ (utils.rs:40), from its LFSR */
    unsigned s = 0xFF;
    for (size_t k = 0; k < i; ++k) s = ((s << 1) | (__builtin_popcount(s & 0xB8u) & 1u)) & 0xFFu;
    return (uint8_t)s;
}

void orc_lora_whitening(uint8_t out[255]) {
    for (size_t i = 0; i < 255; ++i) out[i] = whitening_seq(i);
}

static size_t my_modulo(long v1, size_t v2) { /* utils.rs:966-972 */
    return v1 >= 0 ? (size_t)v1 % v2 : (size_t)((long)v2 + (v1 % (long)v2)) % v2;
}

static uint16_t crc16(uint16_t crc, uint8_t byte_in) { /* encoder.rs:105-117 */
    uint16_t b = byte_in;
    for (int i = 0; i < 8; ++i) {
        if ((((crc & 0x8000) >> 8) ^ (b & 0x80)) != 0) crc = (uint16_t)((crc << 1) ^ 0x1021);
        else crc = (uint16_t)(crc << 1);
        b = (uint16_t)(b << 1);
    }
    return crc;
}

/* Encoder::encode; returns the symbol count, or -1 where the reference panics (> 255 bytes, or < 2 with CRC) */
long orc_lora_encode(int sf, int cr, int has_crc, int ldro, int implicit, const uint8_t *payload, size_t len,
                     uint16_t *out, size_t cap) {
    if (len > 255 || (has_crc && len < 2)) return -1;
    uint8_t frame[5 + 510 + 4], cw[5 + 510 + 4];
    size_t m = 0;
    if (!implicit) { /* header (encoder.rs:64-103) */
        uint8_t o0 = (uint8_t)(len >> 4), o1 = (uint8_t)(len & 0x0F), o2 = (uint8_t)((cr << 1) | (has_crc ? 1 : 0));
        uint8_t c4 = ((o0 & 8) >> 3) ^ ((o0 & 4) >> 2) ^ ((o0 & 2) >> 1) ^ (o0 & 1);
        uint8_t c3 = ((o0 & 8) >> 3) ^ ((o1 & 8) >> 3) ^ ((o1 & 4) >> 2) ^ ((o1 & 2) >> 1) ^ (o2 & 1);
        uint8_t c2 = ((o0 & 4) >> 2) ^ ((o1 & 8) >> 3) ^ (o1 & 1) ^ ((o2 & 8) >> 3) ^ ((o2 & 2) >> 1);
        uint8_t c1 = ((o0 & 2) >> 1) ^ ((o1 & 4) >> 2) ^ (o1 & 1) ^ ((o2 & 4) >> 2) ^ ((o2 & 2) >> 1) ^ (o2 & 1);
        uint8_t c0 = (o0 & 1) ^ ((o1 & 2) >> 1) ^ ((o2 & 8) >> 3) ^ ((o2 & 4) >> 2) ^ ((o2 & 2) >> 1) ^ (o2 & 1);
        frame[m++] = o0; frame[m++] = o1; frame[m++] = o2; frame[m++] = c4;
        frame[m++] = (uint8_t)(c3 << 3 | c2 << 2 | c1 << 1 | c0);
    }
    for (size_t i = 0; i < len; ++i) { /* whitening (:55-62) */
        frame[m++] = (payload[i] ^ whitening_seq(i)) & 0x0F;
        frame[m++] = (payload[i] ^ whitening_seq(i)) >> 4;
    }
    if (has_crc) { /* :119-132 */
        uint16_t crc = 0;
        for (size_t i = 0; i + 2 < len; ++i) crc = crc16(crc, payload[i]);
        crc = crc ^ payload[len - 1] ^ (uint16_t)(payload[len - 2] << 8);
        frame[m++] = crc & 0x000F;
        frame[m++] = (crc & 0x00F0) >> 4;
        frame[m++] = (crc & 0x0F00) >> 8;
        frame[m++] = (crc & 0xF000) >> 12;
    }
    for (size_t i = 0; i < m; ++i) { /* hamming_encode (:134-182) */
        int cr_app = i < (size_t)(sf - (sf < 7 ? 0 : 2)) ? 4 : cr;
        int d0 = (frame[i] >> 3) & 1, d1 = (frame[i] >> 2) & 1, d2 = (frame[i] >> 1) & 1, d3 = frame[i] & 1;
        if (cr_app != 1) {
            int p0 = d3 ^ d2 ^ d1, p1 = d2 ^ d1 ^ d0, p2 = d3 ^ d2 ^ d0, p3 = d3 ^ d1 ^ d0;
            cw[i] = (uint8_t)((d3 << 7 | d2 << 6 | d1 << 5 | d0 << 4 | p0 << 3 | p1 << 2 | p2 << 1 | p3) >> (4 - cr_app));
        } else {
            int p4 = d0 ^ d1 ^ d2 ^ d3;
            cw[i] = (uint8_t)(d3 << 4 | d2 << 3 | d1 << 2 | d0 << 1 | p4);
        }
    }
    size_t cnt = 0, pos = 0, n = 0; /* interleave (:184-268) */
    for (;;) {
        int cw_len, use_ldro;
        if (sf >= 7) {
            cw_len = 4 + (cnt < (size_t)sf - 2 ? 4 : cr);
            use_ldro = cnt < (size_t)sf - 2 || ldro;
        } else {
            cw_len = 4 + (cnt < (size_t)sf ? 4 : cr);
            use_ldro = cnt >= (size_t)sf && ldro;
        }
        size_t sf_app = use_ldro ? (size_t)sf - 2 : (size_t)sf;
        size_t take = m - pos <= sf_app ? m - pos : sf_app;
        uint8_t curr[12] = {0};
        memcpy(curr, cw + pos, take);
        pos += take;
        cnt += sf_app;
        for (int i = 0; i < cw_len; ++i) {
            int inter[12] = {0};
            for (size_t j = 0; j < sf_app; ++j)
                inter[j] = (curr[my_modulo((long)i - (long)j - 1, sf_app)] >> (cw_len - 1 - i)) & 1;
            if (use_ldro) {
                int par = 0;
                for (int j = 0; j < sf; ++j) par += inter[j];
                inter[sf_app] = par % 2 != 0;
            }
            uint16_t v = 0;
            for (int j = 0; j < sf; ++j) v = (uint16_t)(v + (inter[j] << (sf - 1 - j)));
            uint16_t g = v; /* gray_demap (:270-284) */
            for (int j = 1; j < sf; ++j) g ^= (uint16_t)(v >> j);
            if (n < cap) out[n] = (uint16_t)my_modulo((long)g + 1, (size_t)1 << sf);
            ++n;
        }
        if (pos == m) break;
    }
    return (long)n;
}

/* build_upchirp_phase_coherent (utils.rs:917-951) */
void orc_lora_chirp(size_t id, int sf, size_t os, int upchirp, size_t n_samples, int offset_id, float *out) {
    size_t n = (size_t)1 << sf;
    float polarity = upchirp ? 1.0f : -1.0f;
    for (size_t t = 0; t < n_samples; ++t) {
        double t_ds = (double)t / (double)(n * os);
        double tmp = t_ds - 0.5;
        float p = (float)tmp + (float)(offset_id ? (long)id - 1 : (long)id) / (float)n;
        if (p > 0.5f) p -= 1.0f;
        else if (p < -0.5f) p += 1.0f;
        p *= polarity * (1.0f / (float)os) * (2.0f * 3.14159265358979323846f);
        out[t] = p;
    }
}

/* Modulator::modulate + samples_from_phase_diff: writes min(cap, frame length) samples (interleaved re, im) and, when
 * `phase` is not NULL, each sample's phase sum; returns the frame length */
size_t orc_lora_modulate(int sf, size_t os, const uint16_t sync[2], size_t preamble_len, size_t pad,
                         const uint16_t *sym, size_t n_sym, float *out, float *phase, size_t cap) {
    size_t N = ((size_t)1 << sf) * os, Q = N / 4 - os, extra = sf < 7 ? 2 : 0;
    size_t len = 2 * pad + (preamble_len + 4 + extra) * N + Q + n_sym * N;
    static float chirp[1 << 20];
    float last = 0.0f;
    size_t k = 0;
#define EMIT(p_)                                                                                                  \
    do {                                                                                                          \
        float p__ = (p_);                                                                                         \
        if (k < cap) {                                                                                            \
            float th = last + p__, c = cosf(th), s = sinf(th);                                                    \
            out[2 * k] = 1.0f * c - 0.0f * s; /* Complex32::new(1.0, 0.0) * from_polar(1., th) */                 \
            out[2 * k + 1] = 1.0f * s + 0.0f * c;                                                                 \
            if (phase) phase[k] = th;                                                                             \
        }                                                                                                         \
        last += p__;                                                                                              \
        ++k;                                                                                                      \
    } while (0)
    for (size_t i = 0; i < pad; ++i) EMIT(0.0f);
    for (size_t c = 0; c < preamble_len + 5 + extra; ++c) {
        size_t id = 0, ns = N;
        int up = 1;
        if (c < preamble_len) id = 0;
        else if (c == preamble_len) id = sync[0];
        else if (c == preamble_len + 1) id = sync[1];
        else if (c < preamble_len + 4) up = 0;
        else if (c == preamble_len + 4) { up = 0; ns = Q; }
        orc_lora_chirp(id, sf, os, up, ns, 0, chirp);
        for (size_t t = 0; t < ns; ++t) EMIT(chirp[t]);
    }
    for (size_t s = 0; s < n_sym; ++s) {
        orc_lora_chirp(sym[s], sf, os, 1, N, 1, chirp);
        for (size_t t = 0; t < N; ++t) EMIT(chirp[t]);
    }
    for (size_t i = 0; i < pad; ++i) EMIT(0.0f);
#undef EMIT
    return len;
}

/* sample_count (utils.rs:988-1020); -1 where its usize subtraction underflows (a panic in a debug build) */
long long orc_lora_sample_count(int sf, size_t preamble_len, int explicit_header, size_t payload_len, int has_crc,
                                int cr, size_t os, size_t pad, int ldro) {
    float pre = (float)preamble_len + 4.25f + (sf < 7 ? 2.0f : 0.0f);
    size_t hdr = explicit_header ? 5 : 0, pay = 2 * payload_len + (has_crc ? 4 : 0);
    size_t sub = (size_t)sf - (sf >= 7 ? 2 : 0);
    if (pay + hdr < sub) return -1;
    float blocks = ceilf((float)(pay + hdr - sub) / (float)((size_t)sf - (ldro ? 2 : 0)));
    float total = (pre + 8.0f + blocks * (float)(4 + cr)) * (float)(((size_t)1 << sf) * os);
    size_t v = (size_t)total + pad * 2;
    if (v < os) return -1;
    return (long long)(v - os);
}
