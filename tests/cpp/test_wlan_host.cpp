// test_wlan_host.cpp -- the WLAN encoder and Transmitter through the C++ host layer (include/b200sdr.hpp) on a GPU:
// the batch encoder's symbol counts, a stream produced in one exec equals the same stream produced in ragged execs
// across frame boundaries, the burst tags and lengths, the finish rule, reset, and the refusals.  Built by
// __graft_entry__.build(); run by tests/test_gpu_cpp_host.py (needs an H100).
#include <cstdio>
#include <cstring>
#include <vector>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

static std::vector<std::complex<float>> stream(WlanTransmitter &tx, const Instance &inst, size_t cap) {
    const size_t total = (size_t)tx.pending();
    auto *d = inst.device_alloc<std::complex<float>>(total + 1);
    size_t pos = 0;
    while (pos < total) pos += tx.exec(d + pos, cap).first;
    std::vector<std::complex<float>> v(total);
    inst.download(v.data(), d, total);
    inst.device_free(d);
    return v;
}

static size_t burst_len(int32_t mcs, size_t payload, size_t pad_front, size_t pad_tail) {
    size_t ns = 0, nb = 0, np = 0;
    CHECK(b2s_wlan_frame_param(mcs, payload + 28, &ns, &nb, &np) == B2S_OK);
    return pad_front + 320 + 80 * (ns + 1) + (pad_tail > 1 ? pad_tail : 1);
}

int main() {
    Instance inst(0);
    const uint64_t held = b2s_ctx_bytes_held(inst.get());
    const std::array<uint8_t, 6> src{0x42, 0x42, 0x42, 0x42, 0x42, 0x42}, dst{0x23, 0x23, 0x23, 0x23, 0x23, 0x23},
        bss{0xff, 0xff, 0xff, 0xff, 0xff, 0xff};
    {
        const std::vector<size_t> lens = {0, 3, 1500};
        const std::vector<int32_t> mcs = {B2S_WLAN_BPSK_1_2, B2S_WLAN_QAM64_2_3, B2S_WLAN_QAM16_3_4};
        std::vector<uint8_t> bytes(1503, 0x5A);
        uint8_t *d_pay = inst.device_alloc<uint8_t>(bytes.size());
        inst.upload(d_pay, bytes.data(), bytes.size());
        uint8_t *d_sym = inst.device_alloc<uint8_t>(48 * 4096);
        size_t want = 0;
        for (size_t i = 0; i < lens.size(); ++i) {
            size_t ns = 0, nb = 0, np = 0;
            CHECK(b2s_wlan_frame_param(mcs[i], lens[i] + 28, &ns, &nb, &np) == B2S_OK);
            CHECK(nb == ns * (size_t)(mcs[i] == B2S_WLAN_BPSK_1_2 ? 24 : mcs[i] == B2S_WLAN_QAM64_2_3 ? 192 : 144));
            CHECK(np == nb - (16 + 8 * (lens[i] + 28) + 6));
            want += 1 + ns;
        }
        CHECK(wlan_encode(inst, src, dst, bss, 0, 1, d_pay, lens, mcs, d_sym, 4096) == want);
        bool threw = false;
        try { wlan_encode(inst, src, dst, bss, 0, 1, d_pay, lens, mcs, d_sym, want - 1); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);                                   // symbols_cap below the total
        threw = false;
        try { wlan_encode(inst, src, dst, bss, 0, 128, d_pay, lens, mcs, d_sym, 4096); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);                                   // scrambler seed outside 1..127
        inst.sync();
        inst.device_free(d_pay);
        inst.device_free(d_sym);
    }
    {
        const std::vector<std::vector<uint8_t>> frames = {{1, 2, 3, 4}, std::vector<uint8_t>(700, 9), {7, 7, 7}};
        const std::vector<int32_t> mcs = {-1, B2S_WLAN_QAM64_3_4, B2S_WLAN_BPSK_3_4};
        WlanTransmitter a(inst, src, dst, bss, B2S_WLAN_QPSK_1_2, 100, 50);
        WlanTransmitter b(inst, src, dst, bss, B2S_WLAN_QPSK_1_2, 100, 50);
        a.push(frames, mcs);
        b.push(frames, mcs);
        const auto whole = stream(a, inst, (size_t)1 << 30);
        const auto ragged = stream(b, inst, 1237);
        CHECK(whole.size() == ragged.size() && std::memcmp(whole.data(), ragged.data(), whole.size() * 8) == 0);
        CHECK(whole.front() == std::complex<float>(0.0f, 0.0f));   // the front pad
        const auto bursts = a.drain_bursts();
        CHECK(bursts.size() == 3 && bursts[0].index == 0 && bursts[1].index == bursts[0].len &&
              bursts[0].len + bursts[1].len + bursts[2].len == whole.size());
        CHECK(bursts.size() == 3 && bursts[0].len == burst_len(B2S_WLAN_QPSK_1_2, 4, 100, 50) &&
              bursts[1].len == burst_len(B2S_WLAN_QAM64_3_4, 700, 100, 50) &&
              bursts[2].len == burst_len(B2S_WLAN_BPSK_3_4, 3, 100, 50));
        CHECK(a.drain_bursts().empty());
        a.push(frames);
        a.finish();
        a.output.reserve((size_t)a.pending());
        WorkIo io;
        a.work(io);
        CHECK(io.finished && a.pending() == 0);
        a.reset();
        CHECK(a.pending() == 0);
        a.push(frames, mcs);                            // reset is the created state: the same stream again
        const auto again = stream(a, inst, 4096);
        CHECK(again.size() == whole.size() && std::memcmp(again.data(), whole.data(), whole.size() * 8) == 0);
        bool threw = false;
        try { a.push({std::vector<uint8_t>(1501, 0)}); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
        threw = false;
        try { a.push({{1}}, {8}); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
        threw = false;
        try { WlanTransmitter c(inst, src, dst, bss, 8, 0, 0); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
    }
    inst.sync();
    CHECK(b2s_ctx_bytes_held(inst.get()) == held);
    return report();
}
