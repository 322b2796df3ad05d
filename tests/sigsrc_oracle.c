/*
 * sigsrc_oracle.c -- CPU restatement of blocks::SignalSource (src/blocks/signal_source/mod.rs:88-227), its NCO
 * (fxpt_nco.rs:11-43) and FixedPointPhase (fxpt_phase.rs:67-98).  TEST INFRASTRUCTURE ONLY: loaded by
 * tests/sigsrc_oracle.py; the product (futuresdr_b200/ + libb200sdr.so) never links it.
 *
 * Every operation is the reference's, in its order, in f32: compile with -ffp-contract=off so the compiler does not
 * fuse a*b+c, which stable Rust never does.  The sine table is not built here: the caller passes the reference's
 * literals (tests/golden/reference_fxpt_sine_table.json) as table[2 i] = slope, table[2 i + 1] = offset.
 * The reference holds no value-pinning test for this block: parity unpinned, except for the table.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

static const float ORC_PI = 3.14159265358979323846f;   /* std::f32::consts::PI  */
static const float ORC_TAU = 6.28318530717958647692f;  /* std::f32::consts::TAU */

/* Rust `f as i32`: round toward zero, saturate at the i32 range, NaN -> 0 */
static int32_t rust_f32_as_i32(float f) {
    if (isnan(f)) return 0;
    if (f >= 2147483648.0f) return INT32_MAX;
    if (f < -2147483648.0f) return INT32_MIN;
    return (int32_t)f;
}

/* FixedPointPhase::new (fxpt_phase.rs:75-82) */
int32_t orc_fxpt_phase_new(float x) {
    float q = x / ORC_TAU;
    q = q + 0.5f;
    int32_t d = rust_f32_as_i32(floorf(q));
    float df = (float)d;
    float t = df * ORC_TAU;
    float xr = x - t;
    float s = xr * 2147483648.0f;            /* TWO_TO_THE_31 (:72) */
    float v = s / ORC_PI;
    return rust_f32_as_i32(v);
}

/* the builders' increment: FixedPointPhase::new(2.0 * PI * frequency / sample_rate) (mod.rs:130-133) */
int32_t orc_sigsrc_inc(float frequency, float sample_rate) {
    float w = 2.0f * ORC_PI;
    w = w * frequency;
    w = w / sample_rate;
    return orc_fxpt_phase_new(w);
}

/* FixedPointPhase::sin (:85-90) of the wrapped phase word ux; cos (:93-98) passes ux + 0x40000000 */
static float table_eval(const float *table, uint32_t ux) {
    uint32_t index = ux >> 22;               /* WORDBITS - NBITS */
    float frac = (float)(ux & 0x3FFFFFu);    /* ACCUM_MASK */
    float m = table[2 * index] * frac;
    return m + table[2 * index + 1];
}

float orc_fxpt_sin(const float *table, int32_t value) { return table_eval(table, (uint32_t)value); }
float orc_fxpt_cos(const float *table, int32_t value) { return table_eval(table, (uint32_t)value + 0x40000000u); }

/* One SignalSource::work call (mod.rs:88-107) over an output slice of n items: for each item
 * a = phase_to_amplitude(phase); a = a * amplitude; phase += inc (wrapping).
 * wave: 0 cos, 1 sin, 2 square; complex_items selects SignalSourceBuilder<Complex32> (out holds 2 n floats).
 * *phase is the NCO's phase on entry and on return. */
void orc_sigsrc_work(const float *table, int wave, int complex_items, int32_t *phase, int32_t inc, float amplitude,
                     float *out, size_t n) {
    int32_t p = *phase;
    for (size_t k = 0; k < n; k++) {
        if (!complex_items) {
            float a;
            if (wave == 0) a = orc_fxpt_cos(table, p);                       /* mod.rs:134 */
            else if (wave == 1) a = orc_fxpt_sin(table, p);                  /* :147 */
            else a = p < 0 ? 1.0f : 0.0f;                                    /* :161-163 */
            out[k] = a * amplitude;
        } else {
            float re, im;
            if (wave != 2) {                                                 /* cos == sin (:181), (cos, sin) (:195) */
                re = orc_fxpt_cos(table, p);
                im = orc_fxpt_sin(table, p);
            } else {
                int32_t t = p >> 30;                                         /* arithmetic shift (:214) */
                switch (t) {
                    case -2: re = 1.0f; im = 0.0f; break;
                    case -1: re = 1.0f; im = 1.0f; break;
                    case 0: re = 0.0f; im = 1.0f; break;
                    default: re = 0.0f; im = 0.0f; break;                    /* t == 1 */
                }
            }
            out[2 * k] = re * amplitude;                                     /* Complex<f32> * f32 */
            out[2 * k + 1] = im * amplitude;
        }
        p = (int32_t)((uint32_t)p + (uint32_t)inc);                          /* NCO::step, wrapping_add */
    }
    *phase = p;
}
