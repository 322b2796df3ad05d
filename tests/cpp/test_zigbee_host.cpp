// test_zigbee_host.cpp -- the ZigBee ClockRecoveryMm and Decoder through the C++ host layer (include/b200sdr.hpp) on a
// GPU: with omega 1, mu 0 and no gains the clock recovery passes its input through; an out-of-slice step throws
// B2S_ESTATE; a Mac-framed frame laid out as chips decodes to its bytes with a passing FCS, a flipped payload bit fails
// it, ragged execs agree with one exec, reset starts over, and the refusals.  Built by __graft_entry__.build(); run by
// tests/test_gpu_cpp_host.py (needs an H100).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

static const uint32_t kChips[16] = {1618456172u, 1309113062u, 1826650030u, 1724778362u, 778887287u,  2061946375u,
                                    2007919840u, 125494990u,  529027475u,  838370585u,  320833617u,  422705285u,
                                    1368596360u, 85537272u,   139563807u,  2021988657u};

static uint16_t calc_crc(const std::vector<uint8_t> &d) {   // Mac::calc_crc (mac.rs:62-80)
    uint16_t crc = 0;
    for (uint8_t b : d)
        for (int k = 0; k < 8; k++) {
            const uint16_t bit = ((b >> k) & 1u) ^ (crc & 1u);
            crc >>= 1;
            if (bit) crc ^= 0x8408;
        }
    return crc;
}

// the Mac's tx framing (mac.rs:193-220) after the length byte: 9 header bytes, the payload, the FCS (little endian)
static std::vector<uint8_t> body(const std::vector<uint8_t> &payload) {
    std::vector<uint8_t> b = {0x41, 0x88, 0x07, 0xAA, 0x1A, 0xFF, 0xFF, 0x44, 0x33};
    b.insert(b.end(), payload.begin(), payload.end());
    const uint16_t crc = calc_crc(b);
    b.push_back(crc & 0xFF);
    b.push_back(crc >> 8);
    return b;
}

static void symbol(std::vector<float> &x, unsigned s) {       // 32 chips, the first sent in bit 31
    for (int j = 31; j >= 0; j--) x.push_back(((kChips[s] >> j) & 1u) ? 0.75f : -0.5f);
}
static void byte(std::vector<float> &x, uint8_t b) { symbol(x, b & 0xF); symbol(x, b >> 4); }

// `lead` noise-free zero chips, preamble, SFD, length, body, 40 trailing zero chips
static std::vector<float> frame_chips(const std::vector<uint8_t> &b, size_t lead) {
    std::vector<float> x(lead, -1.0f);
    for (int i = 0; i < 8; i++) symbol(x, 0);
    byte(x, 0xA7);
    byte(x, (uint8_t)b.size());
    for (uint8_t v : b) byte(x, v);
    x.insert(x.end(), 40, -1.0f);
    return x;
}

int main() {
    Instance inst(0);
    const uint64_t held = b2s_ctx_bytes_held(inst.get());
    {   // omega 1, mu 0, no gains: every step is one item and mu stays 0, so the outputs are the inputs
        ClockRecoveryMm mm(inst, 1.0f, 0.0f, 0.0f, 0.0f, 0.0f);
        CHECK(mm.look_ahead() == 1);
        std::vector<float> x(100);
        for (size_t i = 0; i < x.size(); i++) x[i] = std::sin(0.3f * (float)i);
        mm.input.set(x);
        mm.output.reserve(200);
        WorkIo io;
        mm.work(io);
        CHECK(io.finished);
        const auto y = mm.output.get();
        CHECK(y.size() == 99 && std::memcmp(y.data(), x.data(), 99 * sizeof(float)) == 0);
    }
    {   // a step of ~3e7 items in an 8-item slice: B2S_ESTATE, nothing consumed past the last in-bounds step
        ClockRecoveryMm mm(inst, 2.0f, 0.000225f, 0.5f, 0.03f, 0.0002f);
        mm.input.set({0.5f, -0.5f, 1e9f, -0.5f, 0.25f, 0.5f, 0.75f, 0.1f});
        mm.output.reserve(100);
        int32_t code = 0;
        try { mm.exec(mm.input.slice(), mm.input.len(), mm.output.slice(), mm.output.capacity()); }
        catch (const Error &e) { code = e.code; }
        CHECK(code == B2S_ESTATE);
    }
    for (float lim : {-0.1f, std::numeric_limits<float>::quiet_NaN()}) {
        bool threw = false;
        try { ClockRecoveryMm bad(inst, 2.0f, 0.1f, 0.5f, 0.1f, lim); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
    }
    {   // one frame decodes to its bytes with a passing FCS; a flipped payload bit fails it
        const std::vector<uint8_t> good = body({'z', 'i', 'g', 'b', 'e', 'e'});
        std::vector<uint8_t> bad = good;
        bad[10] ^= 0x04;
        std::vector<float> x = frame_chips(good, 37);
        const std::vector<float> x2 = frame_chips(bad, 100);
        x.insert(x.end(), x2.begin(), x2.end());
        ZigbeeDecoder d(inst, 6);
        d.input.set(x);
        WorkIo io;
        d.work(io);
        CHECK(io.finished);
        const auto fr = d.drain_frames();
        CHECK(fr.size() == 2);
        if (fr.size() == 2) {
            CHECK(fr[0].len == good.size() && std::memcmp(fr[0].bytes, good.data(), good.size()) == 0 && fr[0].crc_ok == 1);
            CHECK(fr[1].len == bad.size() && std::memcmp(fr[1].bytes, bad.data(), bad.size()) == 0 && fr[1].crc_ok == 0);
            // the completing chip: the last chip of the last byte (lead + 8 preamble + SFD + length + body symbols)
            CHECK(fr[0].index == 37 + 32 * (8 + 2 + 2 + 2 * good.size()) - 1);
        }
        CHECK(d.drain_frames().empty());
        // ragged execs give what one exec gives; reset starts over
        d.reset();
        d.input.set(x);
        size_t pos = 0;
        for (size_t cut : {1u, 33u, 500u, 501u, 700u, 1500u}) pos += d.exec(d.input.slice() + pos, cut - pos);
        pos += d.exec(d.input.slice() + pos, x.size() - pos);
        CHECK(pos == x.size());
        const auto again = d.drain_frames();
        CHECK(again.size() == fr.size());
        for (size_t i = 0; i < std::min(again.size(), fr.size()); i++)
            CHECK(std::memcmp(&again[i], &fr[i], sizeof(b2s_zigbee_frame)) == 0);
    }
    inst.sync();
    CHECK(b2s_ctx_bytes_held(inst.get()) == held);
    return report();
}
