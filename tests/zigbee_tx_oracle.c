// zigbee_tx_oracle.c -- CPU oracle of the ZigBee transmitter (TEST INFRASTRUCTURE ONLY): the chain of
// examples/zigbee/src/bin/tx.rs:37-56 restated one work() call at a time.
//   Mac::tx (mac.rs:135-167): a Blob over MAX_FRAME_SIZE - 11 = 116 bytes is dropped, the others are queued.  The
//     queue's MAX_FRAMES = 128 bound is not restated: whether it bites depends on the scheduler, and the library never
//     drops for queue length (DESIGN §4.21).
//   Mac::work (mac.rs:193-252): pops a frame into current_frame when idle (sequence number taken and incremented then),
//     tags its first byte with Tag::Id(n + 16), and copies it into the output slice.
//   modulator (modulator.rs:4-342): ApplyIntoIter (src/blocks/applyintoiter.rs) of make_nibble(low) then
//     make_nibble(high), 128 Complex32 per byte, each DSSS[nib][c] * SHAPE[k % 4] in f32; an input tag moves to the
//     first output of its byte.
//   IqDelay::work (iq_delay.rs:57-139) with a given PADDING: Tail(0) -> Front(pad, id * 128) at each tagged byte,
//     emitting the burst_start tag 2 pad + id * 128 + 2; Copy delays Q by two samples; Tail(pad) pads.
// The DSSS table is generated from the IEEE 802.15.4 chip sequences of symbols 0 and 8 (cyclic shifts by 4 chips, even
// chips on I, odd on Q); tests/test_zigbee_tx_reference.py holds it to the reference's literals.
// Buffers between the blocks have given capacities; a run() call repeats Mac, modulator, IqDelay work() calls until
// the output slice is full or a round moves nothing.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MAX_FRAME_SIZE 127

static const float SHAPE[4] = {0.0f, 0.70710677f, 1.0f, 0.70710677f};
static const char *CHIPS0 = "11011001110000110101001000101110";
static const char *CHIPS8 = "10001100100101100000011101111011";

typedef struct { uint64_t index, value; } tag_t;

typedef struct {
    size_t pad;
    float dsss[16][16][2];
    // Mac
    uint8_t *q;                    // queued payloads, back to back
    size_t *qlen, qn, qcap, qhead, qoff, qbytes, qbcap;
    uint8_t frame[256];
    uint8_t seq;
    size_t cur_index, cur_len;
    // Mac -> modulator
    uint8_t *b1;
    size_t c1, n1, nt1;
    tag_t *t1;
    // modulator
    float it[128][2];
    size_t it_pos, it_len;
    // modulator -> IqDelay
    float *b2;
    size_t c2, n2, nt2;
    tag_t *t2;
    // IqDelay
    int state;                     // 0 Front(left, size), 1 Copy(left), 2 Tail(left)
    size_t left, size;
    float buf[2];
    size_t buf_n;                  // VecDeque<f32> of at most 2: buf[0] is the front
    uint64_t moved;                // items the blocks have moved so far (a round that moves none ends run())
} zbtx;

void orc_zbtx_dsss(float *out) {   // [16][16][2]
    for (int s = 0; s < 16; ++s) {
        const char *base = s < 8 ? CHIPS0 : CHIPS8;
        const int k = 4 * (s % 8);
        for (int c = 0; c < 16; ++c) {
            const int ci = (2 * c - k + 32) % 32, cq = (2 * c + 1 - k + 32) % 32;   // cyclic shift right by k chips
            out[(s * 16 + c) * 2] = base[ci] == '1' ? 1.0f : -1.0f;
            out[(s * 16 + c) * 2 + 1] = base[cq] == '1' ? 1.0f : -1.0f;
        }
    }
}

void orc_zbtx_shape(float *out) { memcpy(out, SHAPE, sizeof SHAPE); }

void *orc_zbtx_new(size_t pad, size_t c1, size_t c2) {
    zbtx *s = calloc(1, sizeof(zbtx));
    s->pad = pad;
    orc_zbtx_dsss(&s->dsss[0][0][0]);
    const uint8_t hdr[14] = {0x00, 0x00, 0x00, 0xa7, 0x00, 0x41, 0x88, 0x00, 0xaa, 0x1a, 0xff, 0xff, 0x44, 0x33};
    memcpy(s->frame, hdr, sizeof hdr);                  // Mac::new (mac.rs:34-47)
    s->c1 = c1;
    s->c2 = c2;
    s->b1 = malloc(c1);
    s->t1 = malloc((c1 + 1) * sizeof(tag_t));
    s->b2 = malloc(c2 * 2 * sizeof(float));
    s->t2 = malloc((c2 + 1) * sizeof(tag_t));
    s->state = 2;                                       // State::Tail(0)
    return s;
}

void orc_zbtx_free(void *p) {
    zbtx *s = p;
    free(s->q); free(s->qlen); free(s->b1); free(s->t1); free(s->b2); free(s->t2);
    free(s);
}

static uint16_t calc_crc(const uint8_t *d, size_t n) {   // mac.rs:62-80
    uint16_t crc = 0;
    for (size_t i = 0; i < n; ++i)
        for (int k = 0; k < 8; ++k) {
            const int bit = (d[i] & (1 << k)) ? 1 ^ (crc & 1) : (crc & 1);
            crc >>= 1;
            if (bit) crc ^= (1 << 15) ^ (1 << 10) ^ (1 << 3);
        }
    return crc;
}

// Mac::tx with a Blob: 1 if queued, 0 if dropped
int orc_zbtx_tx(void *p, const uint8_t *data, size_t n) {
    zbtx *s = p;
    if (n > MAX_FRAME_SIZE - 11) return 0;
    if (s->qn == s->qcap) {
        s->qcap = s->qcap ? 2 * s->qcap : 64;
        s->qlen = realloc(s->qlen, s->qcap * sizeof(size_t));
    }
    if (s->qbytes + n > s->qbcap) {
        while (s->qbytes + n > s->qbcap) s->qbcap = s->qbcap ? 2 * s->qbcap : 4096;
        s->q = realloc(s->q, s->qbcap);
    }
    memcpy(s->q + s->qbytes, data, n);
    s->qbytes += n;
    s->qlen[s->qn++] = n;
    return 1;
}

static void mac_work(zbtx *s) {
    for (;;) {
        uint8_t *out = s->b1 + s->n1;
        const size_t olen = s->c1 - s->n1;
        if (olen == 0) break;
        if (s->cur_len == 0) {
            if (s->qhead == s->qn) break;
            const size_t n = s->qlen[s->qhead];
            const uint8_t *v = s->q + s->qoff;
            s->qhead++;
            s->qoff += n;
            s->frame[4] = (uint8_t)(n + 11);
            s->frame[7] = s->seq;
            s->seq = (uint8_t)(s->seq + 1);
            memcpy(s->frame + 14, v, n);
            const uint16_t crc = calc_crc(s->frame + 5, 9 + n);
            s->frame[14 + n] = (uint8_t)(crc & 0xff);
            s->frame[15 + n] = (uint8_t)(crc >> 8);
            s->cur_len = n + 16;
            s->cur_index = 0;
            s->t1[s->nt1++] = (tag_t){s->n1, s->cur_len};   // tags.add_tag(0, Tag::Id(len))
            s->moved++;
        } else {
            size_t n = olen < s->cur_len - s->cur_index ? olen : s->cur_len - s->cur_index;
            memcpy(out, s->frame + s->cur_index, n);
            s->n1 += n;
            s->moved += n;
            s->cur_index += n;
            if (s->cur_index == s->cur_len) s->cur_len = 0;
        }
    }
}

static const tag_t *find_tag(const tag_t *t, size_t nt, uint64_t index) {
    for (size_t i = 0; i < nt; ++i)
        if (t[i].index == index) return &t[i];
    return NULL;
}

// drop the first k items (and their tags) of a buffer
static void consume_u8(uint8_t *b, size_t *n, tag_t *t, size_t *nt, size_t k) {
    memmove(b, b + k, *n - k);
    *n -= k;
    size_t j = 0;
    for (size_t i = 0; i < *nt; ++i)
        if (t[i].index >= k) t[j++] = (tag_t){t[i].index - k, t[i].value};
    *nt = j;
}
static void consume_c32(float *b, size_t *n, tag_t *t, size_t *nt, size_t k) {
    memmove(b, b + 2 * k, (*n - k) * 2 * sizeof(float));
    *n -= k;
    size_t j = 0;
    for (size_t i = 0; i < *nt; ++i)
        if (t[i].index >= k) t[j++] = (tag_t){t[i].index - k, t[i].value};
    *nt = j;
}

static void mod_work(zbtx *s) {
    const size_t i_len = s->n1, o0 = s->n2, o_len = s->c2 - s->n2;
    size_t consumed = 0, produced = 0;
    while (produced < o_len) {
        if (s->it_pos < s->it_len) {
            s->b2[2 * (o0 + produced)] = s->it[s->it_pos][0];
            s->b2[2 * (o0 + produced) + 1] = s->it[s->it_pos][1];
            s->it_pos++;
            produced++;
        } else if (consumed < i_len) {
            const uint8_t v = s->b1[consumed];
            for (int h = 0; h < 2; ++h) {
                const int nib = h ? v >> 4 : v & 0x0f;
                for (int k = 0; k < 64; ++k) {                 // [x; 4] zipped with SHAPE cycled
                    const float *x = s->dsss[nib][k / 4];
                    s->it[64 * h + k][0] = x[0] * SHAPE[k % 4];
                    s->it[64 * h + k][1] = x[1] * SHAPE[k % 4];
                }
            }
            s->it_pos = 0;
            s->it_len = 128;
            const tag_t *t = find_tag(s->t1, s->nt1, consumed);
            if (t) s->t2[s->nt2++] = (tag_t){o0 + produced, t->value};
            consumed++;
        } else {
            break;
        }
    }
    s->n2 += produced;
    s->moved += consumed + produced;
    consume_u8(s->b1, &s->n1, s->t1, &s->nt1, consumed);
}

// one IqDelay::work into out[0, olen); its output tags at base + index.  Returns -1 on a missing frame tag (panic).
static long iq_work(zbtx *s, float *out, size_t olen, uint64_t base, uint64_t *ti, uint64_t *tv, size_t tcap,
                    size_t *nt) {
    const float *in = s->b2;
    const size_t i_len = s->n2;
    size_t consumed = 0, produced = 0;
    while (produced < olen) {
        if (s->state == 0) {                                  // Front(left, size)
            size_t n = olen - produced < s->left ? olen - produced : s->left;
            for (size_t k = 0; k < n; ++k) out[2 * (produced + k)] = out[2 * (produced + k) + 1] = 0.0f;
            produced += n;
            if (n == s->left) {
                s->state = 1;
                s->left = s->size;
                s->buf[0] = s->buf[1] = 0.0f;
                s->buf_n = 2;
            } else {
                s->left -= n;
            }
        } else if (s->state == 1) {                           // Copy(left)
            if (s->left == 0) {
                if (s->buf_n) {
                    out[2 * produced] = 0.0f;
                    out[2 * produced + 1] = s->buf[0];
                    s->buf[0] = s->buf[1];
                    s->buf_n--;
                    produced++;
                } else {
                    s->state = 2;
                    s->left = s->pad;
                }
            } else if (consumed == i_len) {
                break;
            } else {
                out[2 * produced] = in[2 * consumed];
                out[2 * produced + 1] = s->buf[0];            // pop_front().unwrap()
                s->buf[0] = s->buf[1];
                s->buf[1] = in[2 * consumed + 1];             // push_back(im)
                produced++;
                consumed++;
                s->left--;
            }
        } else {                                              // Tail(left)
            if (s->left == 0 && consumed == i_len) {
                break;
            } else if (s->left == 0) {
                const tag_t *t = find_tag(s->t2, s->nt2, consumed);
                if (!t) return -1;                            // panic!("no frame start tag")
                s->state = 0;
                s->left = s->pad;
                s->size = (size_t)t->value * 2 * 16 * 4;
                if (*nt < tcap) {
                    ti[*nt] = base + produced;
                    tv[*nt] = 2 * s->pad + (size_t)t->value * 2 * 16 * 4 + 2;
                }
                (*nt)++;
            } else {
                size_t n = olen - produced < s->left ? olen - produced : s->left;
                for (size_t k = 0; k < n; ++k) out[2 * (produced + k)] = out[2 * (produced + k) + 1] = 0.0f;
                produced += n;
                s->left -= n;
            }
        }
    }
    consume_c32(s->b2, &s->n2, s->t2, &s->nt2, consumed);
    s->moved += consumed + produced;
    return (long)produced;
}

// Work rounds (Mac, modulator, IqDelay) until cap samples are out at out (interleaved re, im) or a round moves
// nothing.  The output's burst_start tags go to (ti, tv) as absolute stream indices from base (*nt of them; more than
// tcap are counted, not stored).  Returns the samples produced, or -1 on a missing frame tag.
long orc_zbtx_run(void *p, float *out, size_t cap, uint64_t base, uint64_t *ti, uint64_t *tv, size_t tcap, size_t *nt) {
    zbtx *s = p;
    size_t produced = 0;
    *nt = 0;
    while (produced < cap) {
        const uint64_t moved = s->moved;
        mac_work(s);
        mod_work(s);
        const long r = iq_work(s, out + 2 * produced, cap - produced, base + produced, ti, tv, tcap, nt);
        if (r < 0) return -1;
        produced += (size_t)r;
        if (s->moved == moved) break;
    }
    return (long)produced;
}
