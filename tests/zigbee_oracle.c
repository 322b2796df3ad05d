/* CPU oracle of the ZigBee receiver's DC blocker, ClockRecoveryMm, Decoder and Mac::calc_crc (TEST INFRASTRUCTURE ONLY).
 *
 * Each function restates one reference call, statement by statement: orc_zb_dc_block is the closure of
 * examples/zigbee/src/bin/rx.rs:70-73 (after the phase), orc_zb_mm_work one ClockRecoveryMm::work call
 * (clock_recovery_mm.rs:64-97), orc_zb_decoder_work one Decoder::work call (decoder.rs:108-183), orc_zb_calc_crc
 * Mac::calc_crc (mac.rs:62-80).  f32 arithmetic throughout, built with -ffp-contract=off so that nothing is fused. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

/* rx.rs:72-73: iir = (1.0 - alpha) * iir + alpha * phase; phase - iir */
void orc_zb_dc_block(float alpha, float *iir, const float *x, size_t n, float *y) {
    for (size_t i = 0; i < n; i++) {
        *iir = (1.0f - alpha) * *iir + alpha * x[i];
        y[i] = x[i] - *iir;
    }
}

typedef struct {
    float omega, omega_mid, omega_limit, gain_omega, mu, gain_mu, last_sample;
    uint32_t pad;
    uint64_t look_ahead;
} orc_mm;

static uint64_t as_usize(float f) {            /* Rust's saturating float -> usize cast */
    if (!(f > 0.0f)) return 0;
    if (f >= 18446744073709551616.0f) return UINT64_MAX;
    return (uint64_t)f;
}

/* ClockRecoveryMm::new (clock_recovery_mm.rs:28-58) */
void orc_zb_mm_new(orc_mm *m, float omega, float gain_omega, float mu, float gain_mu, float omega_relative_limit) {
    m->look_ahead = as_usize(ceilf(omega + omega * omega_relative_limit + gain_mu));
    m->omega = omega;
    m->omega_mid = omega;
    m->omega_limit = omega * omega_relative_limit;
    m->gain_omega = gain_omega;
    m->mu = mu;
    m->gain_mu = gain_mu;
    m->last_sample = 0.0f;
    m->pad = 0;
}

static float slice(float i) { return i > 0.0f ? 1.0f : -1.0f; }

/* One work() call.  Returns 0, or 1 when a step would move ii past n_in (the reference would over-consume): the state
 * and the counts are then those before that step. */
int orc_zb_mm_work(orc_mm *m, const float *i, size_t n_in, float *o, size_t n_out, size_t *consumed,
                   size_t *produced) {
    size_t ii = 0, oo = 0;
    int err = 0;
    while (m->look_ahead < n_in && ii < n_in - m->look_ahead && oo < n_out) {
        const float out = i[ii] + m->mu * (i[ii + 1] - i[ii]);
        const float mm_val = slice(m->last_sample) * out - slice(out) * m->last_sample;
        float omega = m->omega + m->gain_omega * mm_val;
        float d = omega - m->omega_mid;                       /* f32::clamp: NaN passes */
        if (d < -m->omega_limit) d = -m->omega_limit;
        if (d > m->omega_limit) d = m->omega_limit;
        omega = m->omega_mid + d;
        const float mu = m->mu + (omega + m->gain_mu * mm_val);
        const uint64_t step = as_usize(floorf(mu));
        if (step > n_in - ii) { err = 1; break; }
        o[oo] = out;
        m->last_sample = out;
        m->omega = omega;
        m->mu = mu - floorf(mu);
        ii += step;
        oo += 1;
    }
    *consumed = ii;
    *produced = oo;
    return err;
}

static const uint32_t CHIP_MAPPING[16] = {
    1618456172u, 1309113062u, 1826650030u, 1724778362u, 778887287u, 2061946375u, 2007919840u, 125494990u,
    529027475u,  838370585u,  320833617u,  422705285u,  1368596360u, 85537272u,  139563807u,  2021988657u};

enum { SEARCH = 0, PREAMBLE_FOUND = 1, SEARCH_SFD = 2, SEARCH_HEADER = 3, DECODE = 4 };

typedef struct {
    uint32_t shift_reg, threshold, chip_count, state;
    int32_t byte;                  /* Option<u8>: -1 = None */
    uint32_t len, dlen;
    uint8_t data[128];
} orc_zb;

void orc_zb_decoder_new(orc_zb *d, uint32_t threshold) {
    memset(d, 0, sizeof(*d));
    d->threshold = threshold;
    d->byte = -1;
}

static int matching(const orc_zb *d, int index) {
    return (uint32_t)__builtin_popcount((d->shift_reg & 0x7FFFFFFEu) ^ (CHIP_MAPPING[index] & 0x7FFFFFFEu)) <
           d->threshold;
}

static int decode(uint32_t seq, uint32_t threshold) {      /* Some(i) -> i, None -> -1 */
    uint32_t best = 0;
    int bi = 0;
    for (int i = 0; i < 16; i++) {
        const uint32_t v = (uint32_t)__builtin_popcount((seq & 0x7FFFFFFEu) ^ (CHIP_MAPPING[i] & 0x7FFFFFFEu));
        if (i == 0 || v < best) { best = v; bi = i; }   /* min_by_key keeps the first minimum */
    }
    return best < threshold ? bi : -1;
}

/* One work() call over in[0, n) (all consumed).  Posted frames: idx = pos0 + the item that completed them, their
 * length and bytes (128 per frame), at most cap of them; returns how many were posted. */
size_t orc_zb_decoder_work(orc_zb *d, const float *in, size_t n, uint64_t pos0, uint64_t *idx, uint32_t *lens,
                           uint8_t *bytes, size_t cap) {
    size_t nf = 0;
    for (size_t k = 0; k < n; k++) {
        const float v = in[k];
        if (v > 0.0f) d->shift_reg = (d->shift_reg << 1) | 1u;
        else d->shift_reg <<= 1;
        d->chip_count = (d->chip_count + 1) % 32;
        switch (d->state) {
        case SEARCH:
            if (matching(d, 0)) { d->state = PREAMBLE_FOUND; d->chip_count = 0; }
            break;
        case PREAMBLE_FOUND:
            if (d->chip_count == 0) {
                if (matching(d, 7)) d->state = SEARCH_SFD;
                else if (!matching(d, 0)) d->state = SEARCH;
            }
            break;
        case SEARCH_SFD:
            if (d->chip_count == 0) {
                if (matching(d, 10)) { d->state = SEARCH_HEADER; d->byte = -1; }
                else d->state = SEARCH;
            }
            break;
        case SEARCH_HEADER:
            if (d->chip_count == 0) {
                const int i = decode(d->shift_reg, d->threshold);
                if (i >= 0) {
                    if (d->byte >= 0) {
                        const uint32_t len = ((uint32_t)i << 4) | (uint32_t)d->byte;
                        if (len < 128) { d->state = DECODE; d->len = len; d->dlen = 0; d->byte = -1; }
                        else d->state = SEARCH;
                    } else {
                        d->byte = i;
                    }
                } else {
                    d->state = SEARCH;
                }
            }
            break;
        case DECODE:
            if (d->chip_count == 0) {
                const int i = decode(d->shift_reg, d->threshold);
                if (i >= 0) {
                    if (d->byte >= 0) {
                        const uint8_t cur = (uint8_t)(((uint32_t)i << 4) | (uint32_t)d->byte);
                        if (d->dlen < 128) d->data[d->dlen] = cur;
                        d->dlen++;
                        d->byte = -1;
                        if (d->dlen == d->len) {
                            if (nf < cap) {
                                idx[nf] = pos0 + k;
                                lens[nf] = d->len;
                                memcpy(bytes + 128 * nf, d->data, d->len);
                            }
                            nf++;
                            d->state = SEARCH;
                        }
                    } else {
                        d->byte = i;
                    }
                } else {
                    d->state = SEARCH;
                }
            }
            break;
        }
    }
    return nf;
}

/* Mac::calc_crc */
uint32_t orc_zb_calc_crc(const uint8_t *data, size_t len) {
    uint16_t crc = 0;
    for (size_t i = 0; i < len; i++)
        for (int k = 0; k < 8; k++) {
            const uint16_t bit = (data[i] & (1u << k)) ? (uint16_t)(1u ^ (crc & 1u)) : (uint16_t)(crc & 1u);
            crc >>= 1;
            if (bit) crc ^= (1u << 15) | (1u << 10) | (1u << 3);
        }
    return crc;
}
