// test_keyfob_host.cpp -- the keyfob slicer and Decoder through the C++ host layer (include/b200sdr.hpp) on a GPU: the
// slicer's outputs, a level stream carrying "0110" + 10101111 + 11010101 decodes to one Close code at the flushing
// edge, ragged execs agree with one exec, reset starts over, firdes::lowpass gives the keyfob's 128 taps, and the
// refusals.  Built by __graft_entry__.build(); run by tests/test_gpu_cpp_host.py (needs an H100).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <string>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

// a bit b is appended by the edge ending a period at level b: a long period from level b, a short one first otherwise
static std::vector<uint8_t> levels(const std::string &bits, size_t lead) {
    std::vector<uint8_t> x(lead, 0);
    uint8_t level = 1;
    auto period = [&](size_t w) { x.insert(x.end(), w, level); level ^= 1; };
    for (char ch : bits) {
        const uint8_t b = ch == '1';
        if (level != b) period(73);
        period(146);
    }
    period(20);
    x.insert(x.end(), 5, level);
    return x;
}

int main() {
    Instance inst(0);
    const uint64_t held = b2s_ctx_bytes_held(inst.get());
    {
        const float nan = std::numeric_limits<float>::quiet_NaN(), inf = std::numeric_limits<float>::infinity();
        Apply<float, uint8_t> slice(inst, B2S_OP_SLICE_F32_U8);
        slice.input.set({1.0f, -1.0f, 0.0f, -0.0f, nan, inf, -inf, 1e-45f, -1e-45f});
        slice.output.reserve(16);
        WorkIo io;
        slice.work(io);
        CHECK(io.finished);
        CHECK((slice.output.get() == std::vector<uint8_t>{1, 0, 0, 0, 0, 1, 0, 1, 0}));
    }
    {
        const std::vector<uint8_t> x = levels("0110" "10101111" "11010101", 300);
        KeyfobDecoder d(inst);
        d.input.set(x);
        WorkIo io;
        d.work(io);
        CHECK(io.finished);
        const auto cd = d.drain_codes();
        CHECK(cd.size() == 1);
        if (cd.size() == 1) {
            CHECK(cd[0].n_bits == 16 && cd[0].label == B2S_KEYFOB_CLOSE);
            CHECK(cd[0].bits[0] == 0xAF && cd[0].bits[1] == 0xD5 && cd[0].bits[2] == 0);
            CHECK(cd[0].index == x.size() - 5);           // the edge that ends the 20-item period
        }
        CHECK(d.drain_codes().empty());
        d.reset();
        d.input.set(x);
        size_t pos = 0;
        for (size_t cut : {1u, 63u, 64u, 500u, 501u, 2049u}) pos += d.exec(d.input.slice() + pos, cut - pos);
        pos += d.exec(d.input.slice() + pos, x.size() - pos);
        CHECK(pos == x.size());
        const auto again = d.drain_codes();
        CHECK(again.size() == cd.size());
        for (size_t i = 0; i < std::min(again.size(), cd.size()); i++)
            CHECK(std::memcmp(&again[i], &cd[i], sizeof(b2s_keyfob_code)) == 0);
        size_t c = 0;
        CHECK(b2s_keyfob_exec(nullptr, d.input.slice(), 4, &c) == B2S_EINVAL);
        CHECK(b2s_keyfob_create(nullptr, nullptr) == B2S_EINVAL);
    }
    {
        const auto t = firdes::lowpass(15e3 / 250e3, windows::hamming(128, false));
        CHECK(t.size() == 128 && std::fabs(t[63] - t[64]) == 0.0f && t[63] > 0.1f);
        bool threw = false;
        try { firdes::lowpass(0.5, {1.0, 1.0}); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
    }
    inst.sync();
    CHECK(b2s_ctx_bytes_held(inst.get()) == held);
    return report();
}
