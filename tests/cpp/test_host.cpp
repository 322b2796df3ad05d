// test_host.cpp -- the reference's known-answer tests replayed through the C++ host layer
// (include/b200sdr.hpp) on a GPU.  Each CHECK names the reference test it restates.
// Built by __graft_entry__.build(); run by tests/test_gpu_cpp_host.py (needs an H100).
#include <cmath>
#include <cstdio>
#include <random>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

using CS = ComputationStatus;
static bool eq(const FilterResult &r, size_t c, size_t p, CS s) {
    return std::get<0>(r) == c && std::get<1>(r) == p && std::get<2>(r) == s;
}

int main() {
    Instance inst(0);

    {   // crates/futuredsp/src/fir.rs:283-319 direct_fir_kernel
        FirFilter<float, float> fir(inst, {1.0f, 2.0f, 3.0f});
        CHECK(fir.length() == 3);
        std::vector<float> in{1, 2, 3}, out(3, 0.f);
        CHECK(eq(fir.filter(in, out), 1, 1, CS::InsufficientInput));
        CHECK(out[0] == 10.0f);
        std::vector<float> none;
        CHECK(eq(fir.filter(in, none), 0, 0, CS::InsufficientOutput));
        std::vector<float> in5{1, 2, 3, 4, 5}, out2(2, 0.f);
        CHECK(eq(fir.filter(in5, out2), 2, 2, CS::InsufficientOutput));
        CHECK(out2[0] == 10.0f && out2[1] == 16.0f);
    }
    {   // fir.rs:321-343 terminating_condition
        FirFilter<float, float> fir(inst, {1.0f, 2.0f});
        std::vector<float> in5{1, 2, 3, 4, 5}, in4{1, 2, 3, 4}, out(3);
        CHECK(eq(fir.filter(in5, out), 3, 3, CS::InsufficientOutput));
        CHECK(eq(fir.filter(in4, out), 3, 3, CS::BothSufficient));
    }
    {   // decimating_fir.rs:341-394 decimation_two
        DecimatingFirFilter<float, float> fir(inst, 2, {1.0f, 2.0f, 3.0f});
        std::vector<float> in{0, 1, 2, 3, 4, 5}, out(3, 0.f), out1(1, 0.f);
        CHECK(eq(fir.filter(in, out), 4, 2, CS::InsufficientInput));
        CHECK(out[0] == 10.0f && out[1] == 22.0f);
        CHECK(eq(fir.filter(in, out1), 2, 1, CS::InsufficientOutput));
        std::vector<float> in5{0, 1, 2, 3, 4};
        CHECK(eq(fir.filter(in5, out1), 2, 1, CS::BothSufficient));
    }
    {   // decimating_fir.rs:396-441 decimation_three
        DecimatingFirFilter<float, float> fir(inst, 3, {1.0f, 2.0f, 1.0f});
        std::vector<float> in{0, 1, 2, 3, 4, 5, 6, 7}, out(3, 0.f), in4{0, 1, 2, 3};
        CHECK(eq(fir.filter(in, out), 6, 2, CS::InsufficientInput));
        CHECK(out[0] == 12.0f && out[1] == 24.0f);
        CHECK(eq(fir.filter(in4, out), 0, 0, CS::InsufficientInput));
    }
    {   // polyphase_resampling_fir.rs:174-260
        PolyphaseResamplingFir<float> f(inst, 3, 2, {1, 2, 3, 4, 5, 6});
        std::vector<float> in{1, 2, 3, 4, 5}, out(8, 0.f), out3(3, 0.f);
        CHECK(eq(f.filter(in, out), 2, 3, CS::InsufficientInput));
        CHECK(out[0] == 6.0f && out[1] == 12.0f && out[2] == 16.0f);
        CHECK(eq(f.filter(in, out3), 2, 3, CS::BothSufficient));
        bool threw = false;
        try { PolyphaseResamplingFir<float> bad(inst, 4, 1, {1, 2, 3, 4, 5, 6}); } catch (const Error &) { threw = true; }
        CHECK(threw);                                   // assert!(taps.num_taps().is_multiple_of(interp))
    }
    {   // tests/fir.rs:7-31: VectorSource -> Fir -> VectorSink through the Mocker
        auto fir = FirBuilder::fir<float, float>(inst, {1.0f, 1.0f, 1.0f});
        Mocker m(fir);
        m.input(std::vector<float>{1, 2, 3, 4, 5, 6});
        m.init_output(6);
        WorkIo io = m.run();
        auto v = m.output();
        CHECK(io.finished && v.size() == 4);
        const float want[4] = {6, 9, 12, 15};
        for (size_t i = 0; i < v.size() && i < 4; i++) CHECK(std::fabs(v[i] - want[i]) < 1.1920929e-7f);
    }
    {   // FirBuilder defaults = the reference's designs (src/blocks/fir.rs:154,:201)
        auto d = FirBuilder::decimating<Complex32>(inst, 4);
        CHECK(d.n_taps() == 52);
        auto r = FirBuilder::resampling<Complex32>(inst, 6, 4);
        CHECK(r.n_taps() == 72);
    }
    {   // Complex<f32> 256-tap FIR, host slices, vs a strict-order host loop (fir.rs:77-88 semantics)
        std::mt19937 g(7);
        std::normal_distribution<float> nd;
        std::uniform_real_distribution<float> ud(-1.f, 1.f);
        const size_t n = 200000, nt = 256;
        std::vector<Complex32> x(n), y(n);
        std::vector<float> taps(nt);
        for (auto &v : x) v = Complex32(nd(g), nd(g));
        float l1 = 0, mx = 0;
        for (auto &t : taps) { t = ud(g); l1 += std::fabs(t); }
        for (auto &v : x) mx = std::max(mx, std::abs(v));
        FirFilter<Complex32, float> fir(inst, taps);
        auto r = fir.filter(x, y);
        CHECK(eq(r, n - nt + 1, n - nt + 1, CS::InsufficientInput));
        double worst = 0;
        for (size_t k = 0; k < n - nt + 1; k += 997) {
            float re = 0, im = 0;
            for (size_t t = 0; t < nt; t++) { re = re + x[k + t].real() * taps[nt - 1 - t]; im = im + x[k + t].imag() * taps[nt - 1 - t]; }
            worst = std::max(worst, (double)std::abs(y[k] - Complex32(re, im)));
        }
        CHECK(worst <= 1e-5 * l1 * mx);
        std::printf("c32 256-tap host-slice FIR: algo=%d worst |err| = %.3e (tol %.3e)\n", fir.algo(), worst, 1e-5 * l1 * mx);
    }
    {   // tests/vulkan.rs:56-76 through Apply: x * 12, length preserved
        Apply<float, float> ap(inst, B2S_OP_SCALE_F32, 12.0f);
        std::vector<float> orig(10000);
        std::mt19937 g(1);
        std::uniform_real_distribution<float> ud(0.f, 1.f);
        for (auto &v : orig) v = ud(g);
        Mocker m(ap);
        m.input(orig);
        m.init_output(orig.size());
        WorkIo io = m.run();
        auto v = m.output();
        CHECK(io.finished && v.size() == orig.size());
        for (size_t i = 0; i < v.size(); i++) CHECK(std::fabs(orig[i] * 12.0f - v[i]) < 1.1920929e-7f);
    }
    {   // Fft block: impulse -> flat spectrum, shift + normalize (fft.rs:196-210)
        Fft fft(inst, 4096, FftDirection::Forward, true, true, 0.5f);
        std::vector<Complex32> x(4096 * 2, Complex32(0, 0));
        x[0] = Complex32(1, 0); x[4096 + 1] = Complex32(1, 0);
        Mocker m(fft);
        m.input(x);
        m.init_output(x.size());
        WorkIo io = m.run();
        auto X = m.output();
        CHECK(io.finished && X.size() == x.size());
        for (size_t k = 0; k < 4096; k += 333) CHECK(std::abs(X[k] - Complex32(0.5f, 0.f)) < 1e-6f);
        // second frame: delta at n=1 -> 0.5*exp(-2 pi i k'/N) with k' = (k + N/2) % N
        for (size_t k = 0; k < 4096; k += 333) {
            const double kp = (double)((k + 2048) % 4096), a = -2.0 * M_PI * kp / 4096.0;
            CHECK(std::abs(X[4096 + k] - Complex32((float)(0.5 * std::cos(a)), (float)(0.5 * std::sin(a)))) < 1e-5f);
        }
    }
    {   // futuredsp::Rotator (rotator.rs:23-48): phase_n = phase_{n-1} * incr THEN out[n] = in[n] * phase_n, un-normalised f32
        const size_t n = 5000;
        const float w = 0.1f;
        std::vector<Complex32> x(n, Complex32(1.0f, -0.5f)), y(n);
        Rotator rot(inst, w);
        Complex32 *dx = inst.device_alloc<Complex32>(n), *dy = inst.device_alloc<Complex32>(n);
        inst.upload(dx, x.data(), n);
        auto r1 = rot.rotate_device(dx, 3000, dy, 3000);                 // two calls: the phase carries over
        auto r2 = rot.rotate_device(dx + 3000, n - 3000, dy + 3000, n);
        CHECK(r1.first == 3000 && r2.first == n - 3000);
        inst.download(y.data(), dy, n);
        float pr = 1.0f, pi = 0.0f;
        const float ir = std::cos(w), ii = std::sin(w);
        double worst = 0;
        for (size_t k = 0; k < n; k++) {
            const float a = pr * ir, b = pi * ii, c = pr * ii, d = pi * ir;     // self.phase *= self.phase_incr FIRST (:26, :40)
            pr = a - b; pi = c + d;
            const Complex32 want(x[k].real() * pr - x[k].imag() * pi, x[k].real() * pi + x[k].imag() * pr);
            worst = std::max(worst, (double)std::abs(y[k] - want));
        }
        CHECK(worst <= 2e-6);
        inst.device_free(dx); inst.device_free(dy);
    }
    {   // blocks::XlatingFir (xlating_fir.rs:42-126): default design, band-pass taps, decimate by 4, rotate
        const size_t D = 4, n = 20000;
        const float offset = 1000.0f, fs = 48000.0f;
        XlatingFir xl(inst, D, offset, fs);
        CHECK(xl.n_taps() == 52);
        std::mt19937 g(3);
        std::normal_distribution<float> nd;
        std::vector<Complex32> x(n);
        for (auto &v : x) v = Complex32(nd(g), nd(g));
        Mocker m(xl);
        m.input(x);
        m.init_output(n / D + 4);
        WorkIo io = m.run();
        auto y = m.output();
        const auto lp = firdes::kaiser::lowpass(0.25, 0.1, 0.0001);
        const size_t nt = lp.size(), want_n = (n + 1 - nt) / D;
        CHECK(io.finished && nt == 52 && y.size() == want_n);
        const float TAU = 6.28318530717958647692f;
        std::vector<Complex32> bpf(nt);
        for (size_t i = 0; i < nt; i++) {
            const float th = (float)i * TAU * offset / fs;
            bpf[i] = Complex32(std::cos(th) * lp[i], std::sin(th) * lp[i]);
        }
        const float w = -TAU * offset * (float)D / fs;
        Complex32 ph(1.0f, 0.0f);
        const Complex32 inc(std::cos(w), std::sin(w));
        double worst = 0;
        for (size_t k = 0; k < std::min(want_n, y.size()); k++) {
            Complex32 acc(0, 0);
            for (size_t t = 0; t < nt; t++) acc += x[D - 1 + k * D + t] * bpf[nt - 1 - t];       // decimating_fir.rs:80-92
            ph = ph * inc;                                                       // rotator.rs:26: phase advances before use
            worst = std::max(worst, (double)std::abs(y[k] - acc * ph));
        }
        CHECK(worst <= 2e-4);
        std::printf("XlatingFir /4: %zu outputs, worst |err| = %.3e\n", y.size(), worst);
    }
    {   // blocks::MovingAvg (moving_avg.rs:72-115): width 4, decay 0.5, one output chunk every 2 input chunks
        MovingAvg ma(inst, 4, 0.5f, 2);
        std::vector<float> in;
        for (float v : {1.f, 3.f, 5.f, 7.f, 9.f}) for (int k = 0; k < 4; k++) in.push_back(v);
        in.push_back(42.f);                                              // trailing partial chunk is left unconsumed
        Mocker m(ma);
        m.input(in);
        m.init_output(16);
        m.run();
        auto v = m.output();
        CHECK(v.size() == 8);
        for (size_t i = 0; i < v.size() && i < 8; i++) CHECK(v[i] == (i < 4 ? 1.75f : 5.1875f));
        {   // the reference's own known answer (tests/moving_avg.rs:7-19): exact f32 equality
            MovingAvg ref(inst, 3, 0.1f, 3);
            Mocker mr(ref);
            mr.input(std::vector<float>{1.f, 2.f, 3.f, 1.f, 2.f, 3.f, 1.f, 2.f, 3.f});
            mr.init_output(3);
            mr.run();
            auto r = mr.output();
            CHECK(r.size() == 3 && r[0] == 0.271f && r[1] == 0.542f && r[2] == 0.813f);
        }
        bool threw = false;
        try { MovingAvg bad(inst, 4, 1.5f, 2); } catch (const Error &) { threw = true; }
        CHECK(threw);                                                    // assert!((0.0..=1.0).contains(&decay_factor))
    }
    {   // SpectrumPipe: a tone at +N/4 cycles/sample lands in bin N/2 + N/4 after the fftshift; 3 frames -> 1 row
        const size_t N = 64, frames = 6;
        SpectrumPipe sp(inst, N, 0.5f, 3);
        std::vector<Complex32> in(N * frames);
        for (size_t i = 0; i < in.size(); i++) {
            const double ph = 2.0 * 3.14159265358979323846 * 0.25 * (double)i;
            in[i] = Complex32((float)std::cos(ph), (float)std::sin(ph));
        }
        Mocker m(sp);
        m.input(in);
        m.init_output(N * 4);
        m.run();
        auto v = m.output();
        CHECK(v.size() == 2 * N);                                        // 6 frames, one row every 3
        size_t peak = 0;
        for (size_t i = 0; i < N && i < v.size(); i++) if (v[N + i] > v[N + peak]) peak = i;
        CHECK(peak == N / 2 + N / 4);
        // |X|^2 = N^2 at the tone; avg after 6 frames with decay 0.5 = N^2 * (1 - 0.5^6)
        if (v.size() == 2 * N) CHECK(std::fabs(v[N + peak] - (float)(N * N) * (1.0f - 0.015625f)) <= 1e-3f * N * N);
    }
    return report();
}
