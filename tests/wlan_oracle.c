/* CPU oracle of the WLAN transmitter (TEST INFRASTRUCTURE ONLY): a C restatement of examples/wlan/src/mac.rs:85-103
 * (generate_mac_data_frame), encoder.rs:22-131 (Enc, with its persistent buffers), mapper.rs:23-69 and :108-132
 * (generate_signal_field, Mapper::map), the constellations of lib.rs:66-175 and the f32 operations of
 * prefix.rs:57-141.  Prefix takes the inverse FFT's outputs from the caller; orc_wlan_ifft_f64 is an f64 DFT of the same
 * transform.  Compiled with -ffp-contract=off so that every f32 operation rounds as the reference's does.  The
 * reference's only WLAN test asserts nothing, so apart from the tables this parity is unpinned. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MAX_PAYLOAD 1500
#define MAX_PSDU (MAX_PAYLOAD + 28)
#define MAX_ENCODED_BITS ((16 + 8 * MAX_PSDU + 6) * 2 + 288)

static const int N_BPSC[8] = {1, 1, 2, 2, 4, 4, 6, 6};
static const int N_DBPS[8] = {24, 36, 48, 72, 96, 144, 192, 216};
static const int RATE[8] = {0x0d, 0x0f, 0x05, 0x07, 0x09, 0x0b, 0x01, 0x03};

/* the scrambler's output from state 0x7F (POLARITY[i] = 1 - 2 seq[i]) */
void orc_wlan_mseq(uint8_t out[127]) {
    unsigned s = 0x7F;
    for (int i = 0; i < 127; ++i) {
        const unsigned fb = ((s >> 6) ^ (s >> 3)) & 1u;
        out[i] = (uint8_t)fb;
        s = ((s << 1) & 0x7Eu) | fb;
    }
}

uint32_t orc_wlan_crc32(const uint8_t *d, size_t n) {
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; ++i) {
        c ^= d[i];
        for (int k = 0; k < 8; ++k) c = (c & 1u) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    }
    return ~c;
}

typedef struct {
    uint8_t frame[MAX_PSDU];
    uint16_t seq;
    uint8_t seed;
    uint8_t bits[MAX_ENCODED_BITS], scrambled[MAX_ENCODED_BITS];
    uint8_t encoded[2 * MAX_ENCODED_BITS], punctured[2 * MAX_ENCODED_BITS], interleaved[2 * MAX_ENCODED_BITS];
} Tx;

/* Mac::new + Encoder::new: a fresh transmitter (sequence number 0, seed 1, zero bit buffers) */
void *orc_wlan_new(const uint8_t *src, const uint8_t *dst, const uint8_t *bss) {
    Tx *t = calloc(1, sizeof(Tx));
    t->frame[0] = 0x08;
    memcpy(t->frame + 4, src, 6);
    memcpy(t->frame + 10, dst, 6);
    memcpy(t->frame + 16, bss, 6);
    t->seed = 1;
    return t;
}
void orc_wlan_free(void *t) { free(t); }
void orc_wlan_set_state(void *tp, unsigned seq, unsigned seed) {
    Tx *t = tp;
    t->seq = (uint16_t)seq;
    t->seed = (uint8_t)seed;
}

/* generate_mac_data_frame: the PSDU of a payload into psdu; its length, or -1 where the Mac drops the payload */
long orc_wlan_mac(void *tp, const uint8_t *data, size_t len, uint8_t *psdu) {
    Tx *t = tp;
    if (len > MAX_PAYLOAD) return -1;
    const uint16_t sn = (uint16_t)(t->seq << 4);
    t->frame[22] = (uint8_t)sn;
    t->frame[23] = (uint8_t)(sn >> 8);
    t->seq = (uint16_t)((t->seq + 1) % 4096);
    memcpy(t->frame + 24, data, len);
    const uint32_t crc = orc_wlan_crc32(t->frame, len + 24);
    for (int i = 0; i < 4; ++i) t->frame[len + 24 + i] = (uint8_t)(crc >> (8 * i));
    memcpy(psdu, t->frame, len + 28);
    return (long)(len + 28);
}

/* FrameParam::new */
void orc_wlan_frame_param(int mcs, size_t psdu, size_t *n_sym, size_t *n_data_bits, size_t *n_pad) {
    const size_t bits = 16 + 8 * psdu + 6, d = (size_t)N_DBPS[mcs];
    *n_sym = bits / d + (bits % d ? 1 : 0);
    *n_data_bits = *n_sym * d;
    *n_pad = *n_data_bits - bits;
}

/* Enc::encode: 48 n_sym subcarrier bytes of the data symbols into out; returns n_sym */
long orc_wlan_encode(void *tp, const uint8_t *psdu, size_t len, int mcs, uint8_t *out, size_t cap) {
    Tx *t = tp;
    size_t n_sym, nd, npad;
    orc_wlan_frame_param(mcs, len, &n_sym, &nd, &npad);
    if (48 * n_sym > cap) return -1;
    /* generate_bits */
    for (size_t i = 0; i < len; ++i)
        for (int b = 0; b < 8; ++b) t->bits[16 + i * 8 + b] = (uint8_t)((psdu[i] >> b) & 1);
    /* scramble */
    unsigned state = t->seed;
    t->seed = (uint8_t)(t->seed + 1);
    if (t->seed > 127) t->seed = 1;
    for (size_t i = 0; i < nd; ++i) {
        const unsigned fb = ((state & 64) ? 1u : 0u) ^ ((state & 8) ? 1u : 0u);
        t->scrambled[i] = (uint8_t)(fb ^ t->bits[i]);
        state = ((state << 1) & 0x7e) | fb;
    }
    memset(t->scrambled + (nd - npad - 6), 0, 6);
    /* convolutional_encode */
    unsigned st = 0;
    for (size_t i = 0; i < nd; ++i) {
        st = ((st << 1) & 0x7e) | t->scrambled[i];
        t->encoded[2 * i] = (uint8_t)(__builtin_popcount(st & 0155) % 2);
        t->encoded[2 * i + 1] = (uint8_t)(__builtin_popcount(st & 0117) % 2);
    }
    /* puncture */
    size_t o = 0;
    for (size_t i = 0; i < 2 * nd; ++i) {
        int keep = 1;
        if (mcs == 6) keep = i % 4 != 3;
        else if (mcs & 1) keep = !(i % 6 == 3 || i % 6 == 4);
        if (keep) t->punctured[o++] = t->encoded[i];
    }
    /* interleave */
    const int bpsc = N_BPSC[mcs], cbps = 48 * bpsc, s = bpsc / 2 > 1 ? bpsc / 2 : 1;
    int first[288], second[288];
    for (int j = 0; j < cbps; ++j) first[j] = s * (j / s) + ((j + (16 * j / cbps)) % s);
    for (int i = 0; i < cbps; ++i) second[i] = 16 * i - (cbps - 1) * (16 * i / cbps);
    for (size_t i = 0; i < n_sym; ++i)
        for (int k = 0; k < cbps; ++k) t->interleaved[i * cbps + k] = t->punctured[i * cbps + second[first[k]]];
    /* split_symbols */
    for (size_t i = 0; i < 48 * n_sym; ++i) {
        uint8_t v = 0;
        for (int k = 0; k < bpsc; ++k) v |= (uint8_t)(t->interleaved[i * bpsc + k] << k);
        out[i] = v;
    }
    return (long)n_sym;
}

static const int SIGNAL_PATTERN[48] = {0, 3, 6, 9, 12, 15, 18, 21, 24, 27, 30, 33, 36, 39, 42, 45,
                                       1, 4, 7, 10, 13, 16, 19, 22, 25, 28, 31, 34, 37, 40, 43, 46,
                                       2, 5, 8, 11, 14, 17, 20, 23, 26, 29, 32, 35, 38, 41, 44, 47};

void orc_wlan_signal_pattern(int32_t out[48]) {
    for (int i = 0; i < 48; ++i) out[i] = SIGNAL_PATTERN[i];
}

/* generate_signal_field: the 48 BPSK bytes of the SIGNAL symbol */
void orc_wlan_signal(int mcs, size_t len, uint8_t out[48]) {
    uint8_t sig[24] = {0}, enc[48];
    const unsigned rate = (unsigned)RATE[mcs];
    for (int i = 0; i < 4; ++i) sig[i] = (uint8_t)((rate >> (3 - i)) & 1);
    for (int i = 0; i < 12; ++i) sig[5 + i] = (uint8_t)((len >> i) & 1);
    unsigned sum = 0;
    for (int i = 0; i < 17; ++i) sum += sig[i];
    sig[17] = (uint8_t)(sum % 2);
    unsigned st = 0;
    for (int i = 0; i < 24; ++i) {
        st = ((st << 1) & 0x7e) | sig[i];
        enc[2 * i] = (uint8_t)(__builtin_popcount(st & 0155) % 2);
        enc[2 * i + 1] = (uint8_t)(__builtin_popcount(st & 0117) % 2);
    }
    for (int i = 0; i < 48; ++i) out[SIGNAL_PATTERN[i]] = enc[i];
}

/* Modulation::map: levels as f32 products */
void orc_wlan_constellation(int bpsc, float *out /* 2 * 2^bpsc */) {
    const float l16 = 0.31622776601683794f, l64 = 0.1543033499620919f, q = 0.70710678118654752440f;
    const float a16[4] = {-3.0f, 3.0f, -1.0f, 1.0f}, a64[8] = {-7.0f, 7.0f, -1.0f, 1.0f, -5.0f, 5.0f, -3.0f, 3.0f};
    for (int i = 0; i < (1 << bpsc); ++i) {
        float re, im;
        switch (bpsc) {
        case 1: re = i ? 1.0f : -1.0f; im = 0.0f; break;
        case 2: re = (i & 1) ? q : -q; im = (i & 2) ? q : -q; break;
        case 4: re = a16[i & 3] * l16; im = a16[i >> 2] * l16; break;
        default: re = a64[i & 7] * l64; im = a64[i >> 3] * l64; break;
        }
        out[2 * i] = re;
        out[2 * i + 1] = im;
    }
}

/* Mapper::map of one symbol: 64 Complex32 (interleaved re, im) */
void orc_wlan_map(const uint8_t in[48], int bpsc, size_t index, float out[128]) {
    float tab[128];
    uint8_t seq[127];
    orc_wlan_constellation(bpsc, tab);
    orc_wlan_mseq(seq);
    memset(out, 0, 128 * sizeof(float));
    const float pol = seq[index % 127] ? -1.0f : 1.0f;
    const int pilots[3] = {11, 25, 39};
    for (int p = 0; p < 3; ++p) {
        out[2 * pilots[p]] = pol;
        out[2 * pilots[p] + 1] = 0.0f;
    }
    out[2 * 53] = -pol;                 /* -POLARITY: (-p, -0.0) */
    out[2 * 53 + 1] = -0.0f;
    int d = 0;
    for (int c = 6; c < 59; ++c) {
        if (c == 11 || c == 25 || c == 32 || c == 39 || c == 53) continue;
        out[2 * c] = tab[2 * in[d]];
        out[2 * c + 1] = tab[2 * in[d] + 1];
        ++d;
    }
}

/* SYNC_WORDS as generated: see wlan.cu's sync_words() for the rule */
void orc_wlan_sync_words(float out[640]) {
    static const signed char S[64] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, -1, 0, 0, 0, 1, 0, 0, 0, -1, 0, 0, 0, -1, 0,
                                      0, 0, 1, 0, 0, 0, 0, 0, 0, 0, -1, 0, 0, 0, -1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0,
                                      1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0};
    static const signed char L[64] = {0, 0, 0, 0, 0, 0, 1, 1, -1, -1, 1, 1, -1, 1, -1, 1, 1, 1, 1, 1, 1, -1, -1, 1, 1,
                                      -1, 1, -1, 1, 1, 1, 1, 0, 1, -1, -1, 1, 1, -1, 1, -1, 1, -1, -1, -1, -1, -1, 1, 1,
                                      -1, -1, 1, -1, 1, -1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
    const double PI = 3.14159265358979323846264338327950288, c = sqrt(13.0 / 6.0);
    double t[2][64][2];
    for (int w = 0; w < 2; ++w)
        for (int n = 0; n < 64; ++n) {
            double re = 0, im = 0;
            for (int i = 0; i < 64; ++i) {
                const signed char x = w ? L[i] : S[i];
                if (!x) continue;
                const double ang = 2.0 * PI * (double)((((i - 32) * n) % 64 + 64) % 64) / 64.0;
                const double xr = x * (w ? 1.0 : c), xi = x * (w ? 0.0 : c);
                re += xr * cos(ang) - xi * sin(ang);
                im += xr * sin(ang) + xi * cos(ang);
            }
            if (fabs(re) < 1e-9) re = 0;
            if (fabs(im) < 1e-9) im = 0;
            t[w][n][0] = re * sqrt(1.0 / 52.0);
            t[w][n][1] = im * sqrt(1.0 / 52.0);
        }
    for (int n = 0; n < 320; ++n) {
        const double *v = n < 160 ? t[0][n % 64] : t[1][(n - 160 + 32) % 64];
        out[2 * n] = (float)v[0];
        out[2 * n + 1] = (float)v[1];
    }
    out[320] = (float)(0.5 * (t[1][32][0] + t[0][0][0]));
    out[321] = (float)(0.5 * (t[1][32][1] + t[0][0][1]));
}

/* the shifted inverse transform of one mapped symbol in f64: y[n] = sqrt(1/52) sum_k in[(k + 32) % 64] e^{2 pi i kn/64} */
void orc_wlan_ifft_f64(const float in[128], double out[128]) {
    const double PI = 3.14159265358979323846264338327950288;
    for (int n = 0; n < 64; ++n) {
        double re = 0, im = 0;
        for (int k = 0; k < 64; ++k) {
            const double ang = 2.0 * PI * (double)((k * n) % 64) / 64.0;
            const double xr = in[2 * ((k + 32) % 64)], xi = in[2 * ((k + 32) % 64) + 1];
            re += xr * cos(ang) - xi * sin(ang);
            im += xr * sin(ang) + xi * cos(ang);
        }
        out[2 * n] = re * sqrt(1.0 / 52.0);
        out[2 * n + 1] = im * sqrt(1.0 / 52.0);
    }
}

/* Prefix::work for one frame of len OFDM symbols whose transforms are y (64 len Complex32): writes its
 * pad_front + 320 + 80 len + max(pad_tail, 1) samples to out (fresh: the first tail sample is windowed against 0) */
long orc_wlan_prefix(const float *y, size_t len, size_t pad_front, size_t pad_tail, float *out, size_t cap) {
    const size_t tail = pad_tail > 1 ? pad_tail : 1, produce = pad_front + tail + len * 80 + 320;
    if (produce > cap) return -1;
    float sync[640];
    orc_wlan_sync_words(sync);
    memset(out, 0, 2 * produce * sizeof(float));
    memcpy(out + 2 * pad_front, sync, sizeof sync);
    for (size_t k = 0; k < len; ++k) {
        const size_t o = pad_front + 320 + k * 80;
        memcpy(out + 2 * o, y + 2 * (k * 64 + 48), 16 * 2 * sizeof(float));
        memcpy(out + 2 * (o + 16), y + 2 * k * 64, 64 * 2 * sizeof(float));
    }
    const size_t o = pad_front + 320;
    out[2 * o] = 0.5f * (out[2 * o] + sync[2 * 256]);
    out[2 * o + 1] = 0.5f * (out[2 * o + 1] + sync[2 * 256 + 1]);
    for (size_t k = 0; k < len; ++k)
        for (int p = 0; p < 2; ++p)
            out[2 * (o + (k + 1) * 80) + p] = 0.5f * (out[2 * (o + (k + 1) * 80) + p] + out[2 * (o + k * 80 + 16) + p]);
    for (size_t i = 0; i < 2 * produce; ++i) out[i] *= 0.6f;
    return (long)produce;
}
