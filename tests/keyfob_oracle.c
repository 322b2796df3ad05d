/* keyfob_oracle.c -- CPU oracle of the keyfob receiver (examples/keyfob/src/{main.rs,decoder.rs}), TEST
 * INFRASTRUCTURE ONLY.  Each function restates one reference call: the running-average closure (main.rs:62-68), the
 * slicer closure (main.rs:73-75) and Decoder::work (decoder.rs:64-127) with Decoder::print (:36-52).  Built with
 * -ffp-contract=off so that f32 products and sums are rounded one by one, as in Rust. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* main.rs:62-68: cur = cur * alpha_inv + x * alpha; x - cur, alpha_inv = 1.0 - alpha, all f32 */
void orc_kf_avg(float alpha, float *cur, const float *x, size_t n, float *y) {
    const float alpha_inv = 1.0f - alpha;
    float c = *cur;
    for (size_t i = 0; i < n; i++) {
        c = c * alpha_inv + x[i] * alpha;
        y[i] = x[i] - c;
    }
    *cur = c;
}

/* main.rs:73-75 */
void orc_kf_slice(const float *x, size_t n, uint8_t *y) {
    for (size_t i = 0; i < n; i++) y[i] = x[i] > 0.0f ? 1 : 0;
}

typedef struct {
    uint64_t n_read;
    uint64_t since;     /* State::Up(since) / State::Down(since) */
    uint32_t up;
    uint32_t output;
    char *s;            /* output_string */
    size_t len, cap;
} orc_kf_dec;

typedef struct {
    uint64_t index;
    uint32_t n_bits;
    int32_t label;
    uint8_t bits[32];
} orc_kf_code;

void orc_kf_dec_new(orc_kf_dec *d) { memset(d, 0, sizeof(*d)); }   /* Down(0), output false, "" */
void orc_kf_dec_free(orc_kf_dec *d) { free(d->s); memset(d, 0, sizeof(*d)); }

static void push(orc_kf_dec *d, char c) {
    if (d->len + 1 >= d->cap) {
        d->cap = d->cap ? 2 * d->cap : 256;
        d->s = (char *)realloc(d->s, d->cap);
    }
    d->s[d->len++] = c;
}

static int ends_with(const char *s, size_t l, const char *t) { return l >= 8 && memcmp(s + l - 8, t, 8) == 0; }

/* decoder.rs:36-52: strip up to the first "10101111" (all of it if there is none); log if >= 8 bits remain */
static size_t print(orc_kf_dec *d, uint64_t index, orc_kf_code *out, size_t n_out, size_t cap) {
    size_t off = d->len;
    for (size_t i = 0; i + 8 <= d->len; i++)
        if (memcmp(d->s + i, "10101111", 8) == 0) { off = i; break; }
    const char *s = d->s + off;
    const size_t l = d->len - off;
    d->len = 0;                                   /* std::mem::take */
    if (l < 8) return n_out;
    if (n_out >= cap) return n_out + 1;
    orc_kf_code *c = out + n_out;
    memset(c, 0, sizeof(*c));
    c->index = index;
    c->n_bits = l > 0xFFFFFFFFu ? 0xFFFFFFFFu : (uint32_t)l;
    c->label = ends_with(s, l, "11010101") ? 1 : ends_with(s, l, "11100011") ? 2 : ends_with(s, l, "10111001") ? 3 : 0;
    for (size_t i = 0; i < l && i < 256; i++)
        if (s[i] == '1') c->bits[i / 8] |= (uint8_t)(0x80u >> (i % 8));
    return n_out + 1;
}

/* decoder.rs:64-127, one call over in[0, n): returns the number of codes logged (those past cap are dropped) */
size_t orc_kf_dec_work(orc_kf_dec *d, const uint8_t *in, size_t n, orc_kf_code *out, size_t cap) {
    size_t n_out = 0;
    for (size_t i = 0; i < n; i++) {
        const uint64_t pos = d->n_read + i;
        if ((!d->up && in[i] == 1) || (d->up && in[i] == 0)) {
            const uint64_t diff = pos - d->since;
            const char bit = d->up ? '1' : '0';   /* falling edge "1", rising "0" */
            if (diff >= 63 && diff <= 83) {
                if (!d->output) {
                    d->output = 1;
                } else {
                    d->output = 0;
                    push(d, bit);
                }
            } else if (diff >= 131 && diff <= 161) {
                d->output = 0;
                push(d, bit);
            } else {
                n_out = print(d, pos, out, n_out, cap);
            }
            d->up = !d->up;
            d->since = pos;
        }
    }
    d->n_read += n;
    return n_out;
}
