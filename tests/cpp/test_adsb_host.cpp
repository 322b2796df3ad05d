// test_adsb_host.cpp -- the ADS-B detector / demodulator / CRC block through the C++ host layer (include/b200sdr.hpp)
// on a GPU: a public DF17 frame laid out as ideal PPM decodes to its bytes, a one-bit error is dropped or forwarded as
// forward_failed_crc says, the repeated-index rule of the detector, ragged execs agree with one exec, and the
// refusals.  Built by __graft_entry__.build(); run by tests/test_gpu_cpp_host.py (needs an H100).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

static const uint8_t kFrame[14] = {0x8D, 0x48, 0x40, 0xD6, 0x20, 0x2C, 0xC3, 0x71, 0xC3, 0x2C, 0xE0, 0x57, 0x60, 0x98};

struct Streams { std::vector<float> s, nf, corr; };

// one preamble at `at` (2 samples per half-symbol, pulses in half-symbols 0, 2, 7, 9) followed by the 112 bits of
// `frame` (bit 1: high first half), and a single trigger at `at`
static Streams ppm(size_t n, size_t at, const uint8_t *frame) {
    Streams st{std::vector<float>(n, 0.0f), std::vector<float>(n, 1.0f), std::vector<float>(n, 0.0f)};
    for (int h : {0, 2, 7, 9}) st.s[at + 2 * h] = st.s[at + 2 * h + 1] = 1.0f;
    for (int b = 0; b < 112; b++) {
        const bool one = (frame[b / 8] >> (7 - b % 8)) & 1;
        const size_t p = at + 32 + 4 * b + (one ? 0 : 2);
        st.s[p] = st.s[p + 1] = 1.0f;
    }
    st.corr[at] = 11.0f;
    return st;
}

static void load(AdsbDemod &d, const Streams &st) {
    d.in_samples.set(st.s);
    d.in_nf.set(st.nf);
    d.in_preamble_cor.set(st.corr);
}

int main() {
    Instance inst(0);
    const uint64_t held = b2s_ctx_bytes_held(inst.get());
    {   // a DF17 frame decodes to its bytes and passes the CRC
        AdsbDemod d(inst, 10.0f);
        load(d, ppm(2000, 300, kFrame));
        WorkIo io;
        d.work(io);
        CHECK(io.finished);
        const auto dets = d.drain_detections();
        const auto pks = d.drain_packets();
        CHECK(dets.size() == 1 && dets[0].index == 300 && dets[0].value == 11.0f);
        CHECK(pks.size() == 1);
        if (pks.size() == 1) {
            CHECK(pks[0].preamble_index == 300 && pks[0].crc_passed == 1 && pks[0].preamble_correlation == 11.0f);
            CHECK(std::memcmp(pks[0].bytes, kFrame, 14) == 0);
        }
        CHECK(d.drain_packets().empty() && d.drain_detections().empty());   // drained lists are empty
    }
    {   // one flipped bit: dropped by Decoder::new(false), forwarded as failed by forward_failed_crc
        uint8_t bad[14];
        std::memcpy(bad, kFrame, 14);
        bad[6] ^= 0x10;
        for (bool fwd : {false, true}) {
            AdsbDemod d(inst, 10.0f, fwd);
            load(d, ppm(2000, 300, bad));
            WorkIo io;
            d.work(io);
            const auto pks = d.drain_packets();
            CHECK(d.drain_detections().size() == 1);
            CHECK(pks.size() == (fwd ? 1u : 0u));
            if (fwd && pks.size() == 1) CHECK(pks[0].crc_passed == 0 && std::memcmp(pks[0].bytes, bad, 14) == 0);
        }
    }
    {   // a trigger whose window peaks at t0 + 31, which triggers again: two tags with the same index
        Streams st{std::vector<float>(300, 0.0f), std::vector<float>(300, 1.0f), std::vector<float>(300, 0.0f)};
        st.corr[10] = 11.0f;
        st.corr[41] = 40.0f;
        for (int h : {0, 2, 7, 9}) st.s[41 + 2 * h] = st.s[41 + 2 * h + 1] = 1.0f;
        AdsbDemod d(inst, 10.0f);
        load(d, st);
        WorkIo io;
        d.work(io);
        const auto dets = d.drain_detections();
        CHECK(dets.size() == 2 && dets[0].index == 41 && dets[1].index == 41 && dets[1].value == 40.0f);
        CHECK(d.drain_packets().empty());                                   // 41 + 480 >= 236 produced items
    }
    {   // ragged execs give what one exec gives; reset starts over
        Streams st = ppm(6000, 300, kFrame);
        Streams st2 = ppm(3000, 10, kFrame);
        for (size_t i = 0; i < 3000; i++) {
            st.s[2900 + i] = std::max(st.s[2900 + i], st2.s[i]);
            st.corr[2900 + i] = std::max(st.corr[2900 + i], st2.corr[i]);
        }
        AdsbDemod d(inst, 10.0f);
        load(d, st);
        size_t pos = 0;
        for (size_t cut : {100u, 700u, 701u, 2950u, 3400u, 5000u}) {
            auto [c, done] = d.exec(d.in_samples.slice() + pos, cut - pos, d.in_nf.slice() + pos, cut - pos,
                                    d.in_preamble_cor.slice() + pos, cut - pos, false);
            CHECK(!done);
            pos += c;
        }
        auto [c, done] = d.exec(d.in_samples.slice() + pos, 6000 - pos, d.in_nf.slice() + pos, 6000 - pos,
                                d.in_preamble_cor.slice() + pos, 6000 - pos, true);
        CHECK(done);
        const auto pks = d.drain_packets();
        CHECK(pks.size() == 2 && pks[0].preamble_index == 300 && pks[1].preamble_index == 2910);
        d.reset();
        WorkIo io;
        d.work(io);
        const auto again = d.drain_packets();
        CHECK(again.size() == 2 && again[1].preamble_index == 2910 && std::memcmp(again[1].bytes, kFrame, 14) == 0);
    }
    for (float thr : {std::numeric_limits<float>::quiet_NaN(), std::numeric_limits<float>::infinity(), -1.0f}) {
        bool threw = false;
        try { AdsbDemod bad(inst, thr); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
    }
    inst.sync();
    CHECK(b2s_ctx_bytes_held(inst.get()) == held);
    return report();
}
