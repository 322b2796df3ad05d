/* CPU oracle of the WLAN and M17 receivers' MovingAverage (TEST INFRASTRUCTURE ONLY).
 *
 * A line-by-line restatement of one Kernel::work() call of
 *   examples/wlan/src/moving_average.rs:67-107  (f32 and Complex32, out[i] = sum)
 *   examples/m17/src/moving_average.rs:41-81    (f32, out[i] = sum / 4800.0)
 * Compiled with -ffp-contract=off and without -ffast-math: every operation is one IEEE f32 add, subtract or divide,
 * in the reference's order.  `impl Sum<&f32> for f32` folds from -0.0 (Rust 1.83 and later; the reference's 2024
 * edition needs 1.85); num_complex's `Sum` folds from Complex::zero() = (+0, +0).
 *
 * State: *pad (starts at len - 1).  Returns 0, or -1 for len == 0. */
#include <stddef.h>
#include <stdint.h>

#define MAX_ITER 4000

static size_t min_sz(size_t a, size_t b) { return a < b ? a : b; }
static size_t sat_sub(size_t a, size_t b) { return a > b ? a - b : 0; }

/* items are `w` floats wide (1: f32, 2: Complex32 as (re, im)); has_div only with w == 1 */
static int work(int w, size_t len, int has_div, float div, size_t *pad, const float *input, size_t input_len,
                int input_finished, float *out, size_t out_len, size_t *consumed, size_t *produced,
                int *call_again, int *finished) {
    *consumed = *produced = 0;
    *call_again = *finished = 0;
    if (len == 0) return -1;
    if (*pad > 0) {                                               /* :76-85 */
        size_t m = min_sz(*pad, out_len);
        for (size_t k = 0; k < m * (size_t)w; k++) out[k] = 0.0f;  /* D::zero() */
        *pad -= m;
        *produced = m;
        if (m < out_len) *call_again = 1;
    } else {                                                      /* :86-104 */
        size_t m = min_sz(min_sz(MAX_ITER, sat_sub(input_len + 1, len)), out_len);
        if (m > 0) {
            for (int c = 0; c < w; c++) {                         /* Complex32: the two components are independent */
                float sum = w == 1 ? -0.0f : 0.0f;                /* input[0..len-1].iter().sum() */
                for (size_t k = 0; k < len - 1; k++) sum = sum + input[k * w + c];
                for (size_t i = 0; i < m; i++) {
                    sum += input[(i + len - 1) * w + c];
                    out[i * w + c] = has_div ? sum / div : sum;
                    sum -= input[i * w + c];
                }
            }
            *consumed = m;
            *produced = m;
        }
        if (input_finished && m == sat_sub(input_len + 1, len)) *finished = 1;
    }
    return 0;
}

int orc_boxavg_work_f32(size_t len, int has_div, float div, size_t *pad, const float *input, size_t input_len,
                        int input_finished, float *out, size_t out_len, size_t *consumed, size_t *produced,
                        int *call_again, int *finished) {
    return work(1, len, has_div, div, pad, input, input_len, input_finished, out, out_len, consumed, produced,
                call_again, finished);
}

int orc_boxavg_work_c32(size_t len, size_t *pad, const float *input, size_t input_len, int input_finished,
                        float *out, size_t out_len, size_t *consumed, size_t *produced, int *call_again,
                        int *finished) {
    return work(2, len, 0, 1.0f, pad, input, input_len, input_finished, out, out_len, consumed, produced, call_again,
                finished);
}
