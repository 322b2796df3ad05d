// test_lora_host.cpp -- the LoRa encoder and Transmitter through the C++ host layer (include/b200sdr.hpp) on a GPU:
// the batch encoder's symbol counts, a stream produced in one exec equals the same stream produced in ragged execs
// across frame boundaries, the burst tags, the finish rule, reset, and the refusals.  Built by
// __graft_entry__.build(); run by tests/test_gpu_cpp_host.py (needs an H100).
#include <cstdio>
#include <cstring>
#include <vector>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

static std::vector<std::complex<float>> stream(LoraTransmitter &tx, const Instance &inst, size_t cap) {
    const size_t total = (size_t)tx.pending();
    auto *d = inst.device_alloc<std::complex<float>>(total + 1);
    size_t pos = 0;
    while (pos < total) pos += tx.exec(d + pos, cap).first;
    std::vector<std::complex<float>> v(total);
    inst.download(v.data(), d, total);
    inst.device_free(d);
    return v;
}

int main() {
    Instance inst(0);
    const uint64_t held = b2s_ctx_bytes_held(inst.get());
    {
        const std::vector<size_t> lens = {0, 2, 255};
        std::vector<uint8_t> bytes(257, 0x5A);
        uint8_t *d_pay = inst.device_alloc<uint8_t>(bytes.size());
        inst.upload(d_pay, bytes.data(), bytes.size());
        uint16_t *d_sym = inst.device_alloc<uint16_t>(4096);
        size_t want = 0;
        for (size_t l : lens) {
            size_t n = 0;
            CHECK(b2s_lora_symbol_count(7, 1, 0, 0, 0, l, &n) == B2S_OK);
            want += n;
        }
        CHECK(lora_encode(inst, 7, 1, false, false, false, d_pay, lens, d_sym, 4096) == want);
        bool threw = false;
        try { lora_encode(inst, 7, 1, true, false, false, d_pay, lens, d_sym, 4096); } catch (const Error &) { threw = true; }
        CHECK(threw);                                   // a 0-byte payload with CRC
        inst.sync();
        inst.device_free(d_pay);
        inst.device_free(d_sym);
    }
    {
        const std::vector<std::vector<uint8_t>> frames = {{1, 2, 3, 4}, {9, 8}, {7, 7, 7, 7, 7, 7, 7}};
        LoraTransmitter a(inst, 7, 2, true, false, false, 4, {8, 16}, 8, 5);
        LoraTransmitter b(inst, 7, 2, true, false, false, 4, {8, 16}, 8, 5);
        a.push(frames);
        b.push(frames);
        const auto whole = stream(a, inst, (size_t)1 << 30);
        const auto ragged = stream(b, inst, 1237);
        CHECK(whole.size() == ragged.size() && std::memcmp(whole.data(), ragged.data(), whole.size() * 8) == 0);
        CHECK(whole.front() == std::complex<float>(1.0f, 0.0f));   // the front pad: zero phase
        const auto bursts = a.drain_bursts();
        CHECK(bursts.size() == 3 && bursts[0].index == 0 && bursts[1].index == bursts[0].len &&
              bursts[0].len + bursts[1].len + bursts[2].len == whole.size());
        CHECK(a.drain_bursts().empty());
        a.push(frames);
        a.finish();
        a.output.reserve((size_t)a.pending());
        WorkIo io;
        a.work(io);
        CHECK(io.finished && a.pending() == 0);
        a.reset();
        CHECK(a.pending() == 0);
        bool threw = false;
        try { a.set_sync_word(128, 0); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
        threw = false;
        try { LoraTransmitter c(inst, 5, 1, true, false, false, 4, {24, 32}, 12, 0); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);                                   // SynchWord::Public does not fit SF5
        threw = false;
        try { LoraTransmitter c(inst, 7, 1, true, false, false, 0, {8, 16}, 8, 0); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
    }
    inst.sync();
    CHECK(b2s_ctx_bytes_held(inst.get()) == held);
    return report();
}
