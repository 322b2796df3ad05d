// test_ssb_host.cpp -- the SSB transceiver's device closures through the C++ host layer (include/b200sdr.hpp) on a
// GPU: Mixer<Complex32> (ROTATE_C32) equals Rotator on the same stream, Mixer<float> (WEAVER_F32) and ROTATE_SCALE_C32
// equal a host restatement of the closures bit for bit across ragged execs and a reset, Apply(DIV_C32) and the
// i16 converter on edge values, and the refusals.  Built by __graft_entry__.build(); run by tests/test_gpu_cpp_host.py
// (needs an H100).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <vector>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

// the closures of examples/ssb, one sample at a time on the host (g++ does not contract these on x86-64)
struct HostOsc {
    float sr, si, pr = 1.0f, pi = 0.0f;
    explicit HostOsc(float theta) : sr(1.0f * std::cos(theta)), si(1.0f * std::sin(theta)) {}
    void step() { const float a = pr; pr = pr * sr - pi * si; pi = pi * sr + a * si; }
};

static bool same_bits(const void *a, const void *b, size_t bytes) { return std::memcmp(a, b, bytes) == 0; }

int main() {
    Instance inst(0);
    const uint64_t held = b2s_ctx_bytes_held(inst.get());
    std::vector<Complex32> x(50'000);
    for (size_t i = 0; i < x.size(); i++) x[i] = Complex32(std::sin(0.001f * i) * 3.0f, std::cos(0.0007f * i) - 0.5f);
    const float theta = -1.2640003f;
    {
        Mixer<Complex32> mix(inst, B2S_MIX_ROTATE_C32, theta);
        Rotator rot(inst, theta);
        Complex32 *di = inst.device_alloc<Complex32>(x.size()), *a = inst.device_alloc<Complex32>(x.size()),
                  *b = inst.device_alloc<Complex32>(x.size());
        inst.upload(di, x.data(), x.size());
        size_t pos = 0;
        for (size_t cut : {1u, 8u, 9u, 4106u, 30'000u}) { pos += mix.mix_device(di + pos, cut - pos, a + pos, cut - pos).first; }
        pos += mix.mix_device(di + pos, x.size() - pos, a + pos, x.size() - pos).first;
        CHECK(pos == x.size());
        rot.rotate_device(di, x.size(), b, x.size());
        std::vector<Complex32> ha(x.size()), hb(x.size());
        inst.download(ha.data(), a, x.size());
        inst.download(hb.data(), b, x.size());
        CHECK(same_bits(ha.data(), hb.data(), x.size() * sizeof(Complex32)));
        inst.device_free(di); inst.device_free(a); inst.device_free(b);
    }
    {
        Mixer<float> weaver(inst, B2S_MIX_WEAVER_F32, 0.19634955f, 0.5f);
        weaver.input.set(x);
        weaver.output.reserve(x.size());
        WorkIo io;
        weaver.work(io);
        CHECK(io.finished);
        HostOsc o(0.19634955f);
        std::vector<float> want(x.size());
        for (size_t i = 0; i < x.size(); i++) {
            o.step();
            const float t1 = x[i].real() * o.pr, t2 = x[i].imag() * o.pi;
            want[i] = 0.5f * (t1 + t2);
        }
        const auto got = weaver.output.get();
        CHECK(got.size() == x.size() && same_bits(got.data(), want.data(), x.size() * sizeof(float)));
    }
    {
        Mixer<Complex32> xl(inst, B2S_MIX_ROTATE_SCALE_C32, theta, 0.0001f);
        xl.input.set(x);
        xl.output.reserve(x.size());
        xl.mix_device(xl.input.slice(), 777, xl.output.slice(), 777);
        xl.reset();                                                   // osc back to 1 + 0i
        WorkIo io;
        xl.work(io);
        HostOsc o(theta);
        std::vector<Complex32> want(x.size());
        for (size_t i = 0; i < x.size(); i++) {
            o.step();
            const float vr = x[i].real(), vi = x[i].imag();
            want[i] = Complex32((vr * o.pr - vi * o.pi) * 0.0001f, (vr * o.pi + vi * o.pr) * 0.0001f);
        }
        const auto got = xl.output.get();
        CHECK(got.size() == x.size() && same_bits(got.data(), want.data(), x.size() * sizeof(Complex32)));
    }
    {
        const float inf = std::numeric_limits<float>::infinity(), nan = std::numeric_limits<float>::quiet_NaN();
        const std::vector<Complex32> e = {{1.0f, -3.0f}, {inf, -inf}, {nan, -0.0f}, {2.0f, -2.0f}, {1e-45f, 0.5f}};
        Apply<Complex32, Complex32> div(inst, B2S_OP_DIV_C32, 0.0001f);
        div.input.set(e);
        div.output.reserve(e.size());
        WorkIo io;
        div.work(io);
        const auto d = div.output.get();
        CHECK(d.size() == e.size() && d[0] == Complex32(1.0f / 0.0001f, -3.0f / 0.0001f) && std::isinf(d[1].real()));
        b2s_apply *conv = nullptr;
        CHECK(b2s_apply_create(inst.get(), B2S_OP_C32_TO_I16_IQ, 0.9f, &conv) == B2S_OK);
        Complex32 *di = inst.device_alloc<Complex32>(e.size());
        int16_t *dq = inst.device_alloc<int16_t>(2 * e.size() + 1);
        inst.upload(di, e.data(), e.size());
        size_t c = 0, p = 0;
        CHECK(b2s_apply_exec(conv, di, e.size(), dq + 1, 2 * e.size() - 1, &c, &p) == B2S_OK);   // odd cap, odd start
        CHECK(c == e.size() - 1 && p == 2 * c);
        std::vector<int16_t> q(p);
        inst.download(q.data(), dq + 1, p);
        CHECK((q == std::vector<int16_t>{29490, -32768, 32767, -32768, 0, 0, 32767, -32768}));
        CHECK(b2s_apply_exec(conv, di, e.size(), di, 2 * e.size(), &c, &p) == B2S_EINVAL);   // in place
        b2s_apply_destroy(conv);
        inst.device_free(di); inst.device_free(dq);
    }
    {
        bool threw = false;
        try { Mixer<Complex32> bad(inst, B2S_MIX_WEAVER_F32, 0.1f); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
        b2s_mixer *m = nullptr;
        CHECK(b2s_mixer_create(inst.get(), (b2s_mix_op)3, 0.1f, 1.0f, &m) == B2S_EINVAL && m == nullptr);
        CHECK(b2s_mixer_create(nullptr, B2S_MIX_ROTATE_C32, 0.1f, 1.0f, &m) == B2S_EINVAL);
        size_t c = 0, p = 0;
        CHECK(b2s_mixer_exec(nullptr, nullptr, 0, nullptr, 0, &c, &p) == B2S_EINVAL);
        CHECK(b2s_mixer_reset(nullptr) == B2S_EINVAL);
        b2s_mixer_destroy(nullptr);
    }
    inst.sync();
    CHECK(b2s_ctx_bytes_held(inst.get()) == held);
    return report();
}
