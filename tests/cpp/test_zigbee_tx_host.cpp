// test_zigbee_tx_host.cpp -- the ZigBee Transmitter through the C++ host layer (include/b200sdr.hpp) on a GPU: a stream
// produced in one exec equals the same stream produced in odd-sized execs across frame boundaries, the burst tags and
// lengths, the dropped-payload count, the finish rule, reset, and the refusals.  Built by __graft_entry__.build(); run
// by tests/test_gpu_cpp_host.py (needs an H100).
#include <cstdio>
#include <cstring>
#include <vector>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

static std::vector<std::complex<float>> stream(ZigbeeTransmitter &tx, const Instance &inst, size_t cap) {
    const size_t total = (size_t)tx.pending();
    auto *d = inst.device_alloc<std::complex<float>>(total + 1);
    size_t pos = 0;
    while (pos < total) pos += tx.exec(d + pos, cap).first;
    std::vector<std::complex<float>> v(total);
    inst.download(v.data(), d, total);
    inst.device_free(d);
    return v;
}

static uint64_t frame_len(size_t n, size_t pad) { return 2 * pad + 128 * (n + 16) + 2; }

int main() {
    Instance inst(0);
    const uint64_t held = b2s_ctx_bytes_held(inst.get());
    {
        const std::vector<std::vector<uint8_t>> frames = {{1, 2, 3, 4}, std::vector<uint8_t>(116, 9),
                                                          std::vector<uint8_t>(117, 1), {}, {7, 7, 7}};
        ZigbeeTransmitter a(inst, 1001), b(inst, 1001);
        CHECK(a.push(frames) == 1);                     // the 117-byte payload is dropped, the others queued
        CHECK(b.push(frames) == 1);
        CHECK(a.pending() == frame_len(4, 1001) + frame_len(116, 1001) + frame_len(0, 1001) + frame_len(3, 1001));
        const auto whole = stream(a, inst, (size_t)1 << 30);
        const auto ragged = stream(b, inst, 997);
        CHECK(whole.size() == ragged.size() && std::memcmp(whole.data(), ragged.data(), whole.size() * 8) == 0);
        CHECK(whole.front() == std::complex<float>(0.0f, 0.0f));   // the front pad
        const float z = whole[1001].real();                        // chip 0 of nibble 1 (symbol 0: +1) at SHAPE 0.0
        CHECK(z == 0.0f && !std::signbit(z));
        const auto bursts = a.drain_bursts();
        CHECK(bursts.size() == 4 && bursts[0].index == 0 && bursts[1].index == bursts[0].len &&
              bursts[0].len == frame_len(4, 1001) && bursts[1].len == frame_len(116, 1001) &&
              bursts[2].len == frame_len(0, 1001) && bursts[3].len == frame_len(3, 1001));
        CHECK(bursts.size() == 4 && bursts[3].index + bursts[3].len == whole.size());
        CHECK(a.drain_bursts().empty());
        a.push(frames);
        a.finish();
        a.output.reserve((size_t)a.pending());
        WorkIo io;
        a.work(io);
        CHECK(io.finished && a.pending() == 0);
        a.reset();
        CHECK(a.pending() == 0);
        a.push(frames);                                  // reset is the created state: the same stream again
        const auto again = stream(a, inst, 4096);
        CHECK(again.size() == whole.size() && std::memcmp(again.data(), whole.data(), whole.size() * 8) == 0);
        bool threw = false;
        try { ZigbeeTransmitter c(inst, (size_t)1 << 32); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
        ZigbeeTransmitter d(inst);                       // the reference's padding
        d.push({{0x42}});
        CHECK(d.pending() == frame_len(1, B2S_ZIGBEE_PADDING));
    }
    inst.sync();
    CHECK(b2s_ctx_bytes_held(inst.get()) == held);
    return report();
}
