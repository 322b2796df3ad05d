/* CPU oracle of the ADS-B receiver's PreambleDetector, Demodulator and Decoder::check_crc (TEST INFRASTRUCTURE ONLY).
 *
 * orc_adsb_detect is one PreambleDetector::work call (examples/adsb/src/preamble_detector.rs:65-146), statement by
 * statement, on the slices it is handed; orc_adsb_demod_bits is the bit loop of Demodulator::work for one tag
 * (demodulator.rs:66-86); orc_adsb_check_crc is Decoder::check_crc (decoder.rs:57-73).  f32 arithmetic throughout,
 * built with -ffp-contract=off so that nothing is fused. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#define N_SAMPLES_PER_HALF_SYM 2

/* Returns num_read (what the call consumes and produces); tags (index relative to the slice, max_corr) go to
 * tag_idx / tag_val, at most cap of them, *n_tags their count. */
size_t orc_adsb_detect(float threshold, const float *samples, size_t len_s, const float *nf, size_t len_nf,
                       const float *corr, size_t len_corr, size_t len_out, uint64_t *tag_idx, float *tag_val,
                       size_t cap, size_t *n_tags) {
    size_t samples_to_read = len_s;
    if (len_nf < samples_to_read) samples_to_read = len_nf;
    if (len_corr < samples_to_read) samples_to_read = len_corr;
    if (len_out < samples_to_read) samples_to_read = len_out;
    long long str = (long long)samples_to_read - 2 * 16 * N_SAMPLES_PER_HALF_SYM;
    samples_to_read = str > 0 ? (size_t)str : 0;
    size_t num_read = 0, nt = 0;
    static const int high[4] = {0, 2, 7, 9};
    static const int low[12] = {1, 3, 4, 5, 6, 8, 10, 11, 12, 13, 14, 15};
    while (num_read < samples_to_read) {
        if (corr[num_read] > threshold * nf[num_read]) {
            float max_corr = corr[num_read] / nf[num_read];
            size_t max_corr_idx = num_read;
            for (int i = 1; i < 16 * N_SAMPLES_PER_HALF_SYM; i++) {
                num_read += 1;
                if (corr[num_read] / nf[num_read] > max_corr) {
                    max_corr = corr[num_read] / nf[num_read];
                    max_corr_idx = num_read;
                }
            }
            float hp[4], lp[12];
            for (int k = 0; k < 4; k++) {
                float acc = -0.0f;                                   /* .sum::<f32>() */
                for (int j = 0; j < N_SAMPLES_PER_HALF_SYM; j++)
                    acc = acc + samples[max_corr_idx + high[k] * N_SAMPLES_PER_HALF_SYM + j];
                hp[k] = acc;
            }
            for (int k = 0; k < 12; k++) {
                float acc = -0.0f;
                for (int j = 0; j < N_SAMPLES_PER_HALF_SYM; j++)
                    acc = acc + samples[max_corr_idx + low[k] * N_SAMPLES_PER_HALF_SYM + j];
                lp[k] = acc;
            }
            float min_high = hp[0], max_high = hp[0], max_low = lp[0];   /* reduce(f32::min / f32::max) */
            for (int k = 1; k < 4; k++) { min_high = fminf(min_high, hp[k]); max_high = fmaxf(max_high, hp[k]); }
            for (int k = 1; k < 12; k++) max_low = fmaxf(max_low, lp[k]);
            if (min_high > 0.1f * max_high && max_low < max_high) {
                if (nt < cap) { tag_idx[nt] = max_corr_idx; tag_val[nt] = max_corr; }
                nt++;
            }
        } else {
            num_read += 1;
        }
    }
    *n_tags = nt;
    return num_read;
}

/* the 112 bits of the tag at `index` of `samples` (the caller checks index + 480 < len) */
void orc_adsb_demod_bits(const float *samples, size_t index, uint8_t *bits) {
    static const float one[4] = {1.0f, 1.0f, -1.0f, -1.0f}, zero[4] = {-1.0f, -1.0f, 1.0f, 1.0f};
    for (size_t s = 0; s < 112; s++) {
        const size_t start = index + 8 * 2 * N_SAMPLES_PER_HALF_SYM + s * 2 * N_SAMPLES_PER_HALF_SYM;
        float c0 = 0.0f, c1 = 0.0f;
        for (int i = 0; i < 2 * N_SAMPLES_PER_HALF_SYM; i++) {
            c0 = c0 + samples[start + i] * zero[i];
            c1 = c1 + samples[start + i] * one[i];
        }
        bits[s] = c0 > c1 ? 0 : 1;
    }
}

int orc_adsb_check_crc(const uint8_t *bits_in, size_t len) {
    static const uint8_t poly[25] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 1};
    uint8_t bits[256];
    if (len > 256 || len < 25) return -1;
    for (size_t i = 0; i < len; i++) bits[i] = bits_in[i];
    for (size_t i = 0; i < len - 24; i++)
        if (bits[i] == 1)
            for (size_t j = 0; j < 25; j++) bits[i + j] ^= poly[j];
    unsigned sum = 0;
    for (size_t i = len - 24; i < len; i++) sum += bits[i];
    return sum == 0;
}
