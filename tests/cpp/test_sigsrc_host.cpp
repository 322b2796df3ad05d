// test_sigsrc_host.cpp -- SignalSourceBuilder, SignalSource and Head (src/blocks/signal_source/mod.rs, head.rs) through
// the C++ host layer (include/b200sdr.hpp) on a GPU.  The expected samples come from the host-side FixedPointPhase
// (b2s_fxpt_phase_new / b2s_fxpt_sin_cos): phase k = phase0 + k inc (wrapping), sample = f(phase) * amplitude.
// Built by __graft_entry__.build(); run by tests/test_gpu_cpp_host.py (needs an H100).
#include <cstdio>
#include <cstring>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

static bool same_bits(const void *a, const void *b, size_t bytes) { return std::memcmp(a, b, bytes) == 0; }

int main() {
    Instance inst(0);
    const float fs = 48000.0f, f = 1000.0f, amp = 0.5f, ph0 = 0.25f;
    const FixedPointPhase p0 = FixedPointPhase::make(ph0);
    const FixedPointPhase inc = FixedPointPhase::make(2.0f * 3.14159265358979323846f * f / fs);   // mod.rs:130-133
    auto phase_at = [&](size_t k) {
        FixedPointPhase p;
        p.value = (int32_t)((uint32_t)p0.value + (uint32_t)k * (uint32_t)inc.value);
        return p;
    };
    const size_t n = 5000;
    {   // f32 sin under Mocker, two calls: the second continues the phase
        auto src = SignalSourceBuilder<float>::sin(inst, f, fs, amp, ph0);
        CHECK(src.phase().first.value == p0.value && src.phase().second.value == inc.value);
        Mocker<SignalSource<float>> m(src);
        m.init_output(n);
        WorkIo io = m.run();
        CHECK(!io.finished);
        auto y = m.output();
        CHECK(y.size() == n);
        std::vector<float> want(n);
        for (size_t k = 0; k < n; k++) want[k] = phase_at(k).sin() * amp;
        CHECK(y.size() == n && same_bits(y.data(), want.data(), n * sizeof(float)));
        src.set_amplitude(-1.0f);
        m.init_output(7);
        m.run();
        y = m.output();
        for (size_t k = 0; k < 7; k++) want[k] = phase_at(n + k).sin() * -1.0f;
        CHECK(y.size() == 7 && same_bits(y.data(), want.data(), 7 * sizeof(float)));
        CHECK(src.phase().first.value == phase_at(n + 7).value);
    }
    {   // Complex32 cos is (cos, sin) (mod.rs:175-199); square (value < 0) for f32
        auto c = SignalSourceBuilder<Complex32>::cos(inst, f, fs, amp, ph0);
        Mocker<SignalSource<Complex32>> m(c);
        m.init_output(n);
        m.run();
        auto y = m.output();
        std::vector<Complex32> want(n);
        for (size_t k = 0; k < n; k++) want[k] = Complex32(phase_at(k).cos() * amp, phase_at(k).sin() * amp);
        CHECK(y.size() == n && same_bits(y.data(), want.data(), n * sizeof(Complex32)));
        auto sq = SignalSourceBuilder<float>::square(inst, f, fs, amp, ph0);
        Mocker<SignalSource<float>> ms(sq);
        ms.init_output(n);
        ms.run();
        auto ys = ms.output();
        std::vector<float> ws(n);
        for (size_t k = 0; k < n; k++) ws[k] = (phase_at(k).value < 0 ? 1.0f : 0.0f) * amp;
        CHECK(ys.size() == n && same_bits(ys.data(), ws.data(), n * sizeof(float)));
    }
    {   // Head (head.rs:57-83): min(n_items, input, output); finishes only when n_items reaches 0
        Head<float> h(inst, 10);
        Mocker<Head<float>> m(h);
        m.input(std::vector<float>{1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12});
        m.init_output(4);
        WorkIo io = m.run();
        CHECK(!io.finished && h.n_items() == 6 && m.output() == std::vector<float>({1, 2, 3, 4}));
        m.init_output(100);
        io = m.run();
        CHECK(io.finished && h.n_items() == 0 && m.output() == std::vector<float>({5, 6, 7, 8, 9, 10}));
        Head<float> h2(inst, 100);
        Mocker<Head<float>> m2(h2);
        m2.input(std::vector<float>{1, 2, 3});
        m2.init_output(100);
        io = m2.run();
        CHECK(!io.finished && h2.n_items() == 97);                // the input finished, Head does not
    }
    {   // an invalid wave is refused
        bool refused = false;
        try { SignalSource<float> s(inst, (b2s_wave)3, f, fs, amp, ph0); } catch (const Error &e) { refused = e.code == B2S_EINVAL; }
        CHECK(refused);
    }
    inst.sync();
    return report();
}
