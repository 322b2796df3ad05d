// test_boxavg_host.cpp -- the WLAN / M17 MovingAverage through the C++ host layer (include/b200sdr.hpp) on a GPU: the
// reference's own Mocker known answers (examples/wlan/src/moving_average.rs:117-153), the call loop, a Complex32 case,
// the M17 divisor and the refusals.
// Built by __graft_entry__.build(); run by tests/test_gpu_cpp_host.py (needs an H100).
#include <cmath>
#include <cstdio>
#include <cstring>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

template <typename Block> static WorkIo mocker_run(Block &b) {                     // Mocker::run: again while call_again
    WorkIo io;
    for (int guard = 0; guard < 64; guard++) {
        io = WorkIo{};
        b.work(io);
        if (!io.call_again) break;
    }
    return io;
}

static uint32_t bits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }

int main() {
    Instance inst(0);
    const uint64_t held = b2s_ctx_bytes_held(inst.get());
    {   // mov_avg_one, mov_avg_no_data, mov_avg_data (one reference call per work(), as under Mocker)
        MovingAverage<float> a(inst, 2, std::nullopt, 1);
        a.input.set({1.0f, 2.0f});
        a.output.reserve(2);
        mocker_run(a);
        CHECK(a.output.get() == std::vector<float>({0.0f, 3.0f}));
        MovingAverage<float> b(inst, 3, std::nullopt, 1);
        b.input.set({1.0f, 2.0f});
        b.output.reserve(2);
        mocker_run(b);
        CHECK(b.output.get() == std::vector<float>({0.0f, 0.0f}));
        MovingAverage<float> c(inst, 2, std::nullopt, 1);
        c.input.set({1.0f, 2.0f, 3.0f, 4.0f});
        c.output.reserve(4);
        mocker_run(c);
        CHECK(c.output.get() == std::vector<float>({0.0f, 3.0f, 5.0f, 7.0f}));
    }
    {   // back-to-back calls: 9000 ones, len 5 -> 4 zeros, then runs of 4000, 4000, 996 sums of 5; finished
        MovingAverage<float> a(inst, 5);
        a.input.set(std::vector<float>(9000, 1.0f));
        a.output.reserve(9100);
        WorkIo io;
        a.work(io);
        const std::vector<float> o = a.output.get();
        CHECK(io.finished && !io.call_again && o.size() == 9000);
        bool ok = o.size() == 9000;
        for (size_t i = 0; ok && i < o.size(); i++) ok = o[i] == (i < 4 ? 0.0f : 5.0f);
        CHECK(ok);
    }
    {   // the -0.0 fold, and Complex32 component-wise
        MovingAverage<float> z(inst, 3);
        z.input.set({-0.0f, -0.0f, -0.0f});
        z.output.reserve(3);
        WorkIo io;
        z.work(io);
        const std::vector<float> o = z.output.get();
        CHECK(o.size() == 3 && bits(o[2]) == 0x80000000u);
        MovingAverage<Complex32> c(inst, 2);
        c.input.set({{1, -1}, {2, -2}, {3, -3}});
        c.output.reserve(3);
        c.work(io);
        CHECK(c.output.get() == std::vector<Complex32>({{0, 0}, {3, -3}, {5, -5}}));
    }
    {   // m17: sum / 4800.0, an IEEE division
        MovingAverage<float> m(inst, 2, 4800.0f);
        m.input.set({1.0f, 2.0f});
        m.output.reserve(2);
        WorkIo io;
        m.work(io);
        const std::vector<float> o = m.output.get();
        CHECK(o.size() == 2 && o[1] == 3.0f / 4800.0f);
        m.reset();
        m.input.set({1.0f, 2.0f});
        m.output.reserve(1);
        m.work(io);
        CHECK(m.output.get() == std::vector<float>({0.0f}));
    }
    {   // refusals: len 0, a divisor on Complex32
        bool threw = false;
        try { MovingAverage<float> bad(inst, 0); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
        threw = false;
        try { MovingAverage<Complex32> bad(inst, 48, 4800.0f); } catch (const Error &e) { threw = e.code == B2S_EINVAL; }
        CHECK(threw);
    }
    inst.sync();
    CHECK(b2s_ctx_bytes_held(inst.get()) == held);
    return report();
}
