// firdes.cu -- host-side tap design used by FirBuilder defaults.  f64 math, runs once per
// plan; follows futuredsp::firdes::kaiser::{lowpass,multirate} (crates/futuredsp/src/firdes/
// basic.rs:310-321, :412-459), windows::kaiser (windows.rs:144-152) and besseli0
// (math/special_funs.rs:22-45, Abramowitz & Stegun 9.8.1/9.8.2) so that a graph built with
// FirBuilder::decimating(4) gets the same 52 taps it gets from the reference.
#include <cmath>
#include <vector>

#include "common.cuh"

namespace {
constexpr double kPi = 3.14159265358979323846264338327950288;

double ipow(double x, int n) {              // f64::powi
    const bool recip = n < 0;
    unsigned m = recip ? (unsigned)(-n) : (unsigned)n;
    double r = 1.0;
    for (;;) {
        if (m & 1) r *= x;
        m >>= 1;
        if (!m) break;
        x *= x;
    }
    return recip ? 1.0 / r : r;
}

double bessel_i0(double x) {
    const double t = x / 3.75;
    if (std::fabs(x) <= 3.75) {
        static const double c[6] = {3.5156229, 3.0899424, 1.2067492, 0.2659732, 0.0360768, 0.0045813};
        double s = 1.0;
        for (int i = 0; i < 6; i++) s += c[i] * ipow(t, 2 * (i + 1));
        return s;
    }
    static const double d[9] = {0.39894228, 0.01328592, 0.00225319, -0.00157565, 0.00916281,
                                -0.02057706, 0.02635537, -0.01647633, 0.00392377};
    double s = d[0];
    for (int i = 1; i < 9; i++) s += d[i] * ipow(t, -i);
    return s / (std::sqrt(std::fabs(x)) * std::exp(-x));
}

std::vector<double> kaiser_window(size_t len, double beta) {
    std::vector<double> w(len);
    const double alpha = (double)(len - 1) / 2.0, den = bessel_i0(beta);
    for (size_t n = 0; n < len; n++) {
        const double r = ((double)n - alpha) / alpha;
        w[n] = bessel_i0(beta * std::sqrt(1.0 - r * r)) / den;
    }
    return w;
}

std::vector<double> windowed_sinc(double cutoff, const std::vector<double> &win) {
    const double omega_c = 2.0 * kPi * cutoff, alpha = (double)(win.size() - 1) / 2.0;
    std::vector<double> h(win.size());
    for (size_t n = 0; n < win.size(); n++) {
        const double x = (double)n - alpha;
        h[n] = win[n] * (x == 0.0 ? omega_c / kPi : std::sin(omega_c * x) / (kPi * x));
    }
    return h;
}

double kaiser_beta(double max_ripple) {
    const double a = -20.0 * std::log10(max_ripple);
    if (a > 50.0) return 0.1102 * (a - 8.7);
    if (a >= 21.0) return 0.5842 * std::pow(a - 21.0, 0.4) + 0.07886 * (a - 21.0);
    return 0.0;
}
}  // namespace

extern "C" {

size_t b2s_firdes_kaiser_lowpass(double cutoff, double transition_bw, double max_ripple, float *taps,
                                 size_t cap) {
    if (!(cutoff > 0.0) || !(transition_bw > 0.0) || !(cutoff + transition_bw < 0.5)) return 0;
    const double a = -20.0 * std::log10(max_ripple);
    const size_t n = (size_t)(std::ceil((a - 7.95) / (14.36 * transition_bw)) + 1.0);
    if (!taps || cap < n) return n;
    const auto h = windowed_sinc((2.0 * cutoff + transition_bw) / 2.0, kaiser_window(n, kaiser_beta(max_ripple)));
    for (size_t i = 0; i < n; i++) taps[i] = (float)h[i];
    return n;
}

size_t b2s_firdes_kaiser_multirate(size_t interp, size_t decim, size_t half_polyphase_len,
                                   double max_ripple, float *taps, size_t cap) {
    if (interp == 0 || decim == 0 || half_polyphase_len == 0) return 0;
    if (interp == 1 && decim == 1) {
        if (taps && cap >= 1) taps[0] = 1.0f;
        return 1;
    }
    const size_t band = interp == 1 ? decim : interp, n = 2 * half_polyphase_len * band;
    if (!taps || cap < n) return n;
    auto win = kaiser_window(n + 1, kaiser_beta(max_ripple));
    for (auto &w : win) w *= (double)interp;
    const auto h = windowed_sinc(1.0 / (2.0 * (double)std::max(interp, decim)), win);
    for (size_t i = 0; i < n; i++) taps[i] = (float)h[i];
    return n;
}

// windows::gen_cos (windows.rs:68-94) with coeffs {0.54, 0.46}, literally: alpha is computed in f32 and widened, pi is
// f32::consts::PI widened to f64, and the terms (-1)^k c_k cos(pi (k n) / alpha) are summed in k order.
size_t b2s_window_hamming(size_t len, int32_t periodic, double *out, size_t cap) {
    if (len == 0) return 0;
    if (!out || cap < len) return len;
    static const double coeffs[2] = {0.54, 0.46};
    const size_t npts = periodic ? len + 1 : len;
    const double alpha = (double)((float)(npts - 1) / 2.0f);
    const double pi = (double)3.14159265358979323846f;
    for (size_t n = 0; n < len; n++) {               // the periodic window's extra last point is dropped
        double s = -0.0;
        for (int k = 0; k < 2; k++) {
            const double sign = (k & 1) ? -1.0 : 1.0;  // (-1.0).powi(k)
            s += sign * coeffs[k] * std::cos(pi * (double)(k * n) / alpha);
        }
        out[n] = s;
    }
    return len;
}

// firdes::hilbert (basic.rs:202-222), literally: the odd taps h +- i for i in (1..h).step_by(2), the gain recurrence,
// then x / gain cast to f32.
size_t b2s_firdes_hilbert(const double *window, size_t len, float *taps, size_t cap) {
    if (len == 0 || len % 2 == 0) return 0;
    if (!window || !taps || cap < len) return len;
    std::vector<double> t(len, 0.0);
    const size_t h = (len - 1) / 2;
    double gain = 0.0;
    for (size_t i = 1; i < h; i += 2) {
        const double x = 1.0 / (double)i;
        t[h + i] = x * window[h + i];
        t[h - i] = -x * window[h - i];
        gain = t[h + i] - gain;
    }
    gain = 2.0 * std::fabs(gain);
    for (size_t i = 0; i < len; i++) taps[i] = (float)(t[i] / gain);
    return len;
}

// firdes::lowpass (basic.rs:25-42): window[n] * sinc term, omega_c / pi at x == 0, then cast to f32
size_t b2s_firdes_lowpass(double cutoff, const double *window, size_t len, float *taps, size_t cap) {
    if (len == 0 || !(std::fabs(cutoff) < 0.5)) return 0;
    if (!window || !taps || cap < len) return len;
    const auto h = windowed_sinc(cutoff, std::vector<double>(window, window + len));
    for (size_t i = 0; i < len; i++) taps[i] = (float)h[i];
    return len;
}

}  // extern "C"
