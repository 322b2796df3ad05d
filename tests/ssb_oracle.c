/* ssb_oracle.c -- CPU oracle of the SSB transceiver's closures (examples/ssb/{transmit,receive}.rs), TEST
 * INFRASTRUCTURE ONLY.  Each function restates one Apply / ApplyNM call over a slice, with the closure's state (the
 * oscillator `osc`) carried across calls by the caller:
 *   mixer      transmit.rs:100-107   osc *= shift; v * osc
 *   xlating    receive.rs:58-66      osc *= shift; v * osc * 0.0001
 *   weaver     receive.rs:73-83      osc *= shift; 0.5 * (v.re * osc.re + v.im * osc.im)
 *   file level transmit.rs:125       v * 2.0 / 0.0001
 *   to_i16_iq  transmit.rs:109-112   (re * 0.9 * i16::MAX as f32) as i16, the same of im
 * with shift = Complex32::from_polar(1.0, theta) = (1.0 * cos(theta), 1.0 * sin(theta)).  num_complex's MulAssign and
 * Mul, Complex * f32 and Complex / f32 are written out part by part.  Built with -ffp-contract=off so that every f32
 * product and sum is rounded by itself, as in Rust. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

enum { ROTATE = 0, ROTATE_SCALE = 1, WEAVER = 2 };

void orc_ssb_from_polar(float theta, float *shift) {
    shift[0] = 1.0f * cosf(theta);
    shift[1] = 1.0f * sinf(theta);
}

/* one call of a mixer closure over n samples; osc[2] is the state (1 + 0i initially), out is c32 (2n floats) for
 * ROTATE / ROTATE_SCALE and f32 (n floats) for WEAVER */
void orc_ssb_mix(int op, const float *shift, float param, float *osc, const float *in, size_t n, float *out) {
    const float sr = shift[0], si = shift[1];
    float pr = osc[0], pi = osc[1];
    for (size_t k = 0; k < n; k++) {
        /* MulAssign: re = re * sr - im * si; im = im * sr + re_old * si */
        const float a = pr;
        pr = pr * sr - pi * si;
        pi = pi * sr + a * si;
        const float vr = in[2 * k], vi = in[2 * k + 1];
        if (op == WEAVER) {
            const float term1 = vr * pr;
            const float term2 = vi * pi;
            out[k] = param * (term1 + term2);
        } else {
            /* Mul: (vr pr - vi pi, vr pi + vi pr) */
            float yr = vr * pr - vi * pi;
            float yi = vr * pi + vi * pr;
            if (op == ROTATE_SCALE) { yr = yr * param; yi = yi * param; }
            out[2 * k] = yr;
            out[2 * k + 1] = yi;
        }
    }
    osc[0] = pr;
    osc[1] = pi;
}

/* v * gain / div: Complex * f32 then Complex / f32, each part by itself */
void orc_ssb_file_level(float gain, float div, const float *in, size_t n, float *out) {
    for (size_t k = 0; k < 2 * n; k++) {
        const float t = in[k] * gain;
        out[k] = t / div;
    }
}

/* Rust `f as i16`: truncation toward zero, saturation, NaN -> 0 */
static int16_t as_i16(float f) {
    if (f != f) return 0;
    if (f >= 32767.0f) return 32767;
    if (f <= -32768.0f) return -32768;
    return (int16_t)f;
}

void orc_ssb_to_i16_iq(float level, const float *in, size_t n, int16_t *out) {
    for (size_t k = 0; k < 2 * n; k++) {
        const float t = in[k] * level;
        out[k] = as_i16(t * 32767.0f);
    }
}
