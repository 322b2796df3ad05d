// test_stream_host.cpp -- Combine, Split, Delay, StreamDuplicator, StreamDeinterleaver, firdes::hilbert and
// windows::hamming through the C++ host layer (include/b200sdr.hpp) on a GPU, with the reference's own known answers
// (tests/combine.rs, tests/split.rs, firdes/basic.rs:229-247) and small restated cases.
// Built by __graft_entry__.build(); run by tests/test_gpu_cpp_host.py (needs an H100).
#include <cmath>
#include <cstdio>
#include <cstring>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

template <typename Block> static WorkIo run(Block &b) {
    WorkIo io;
    for (int guard = 0; guard < 64; guard++) {
        io = WorkIo{};
        b.work(io);
        if (io.finished || !io.call_again) break;
    }
    return io;
}

int main() {
    Instance inst(0);
    const uint64_t held = b2s_ctx_bytes_held(inst.get());
    {   // tests/combine.rs:34-57: first input longer; the block finishes on the second input
        Combine<float, float, float> c(inst, B2S_COMBINE_ADD_F32);
        c.in0.set({1, 2, 3, 4, 11, 12});
        c.in1.set({5, 6, 7, 8});
        c.output.reserve(16);
        WorkIo io = run(c);
        CHECK(io.finished && c.output.get() == std::vector<float>({6, 8, 10, 12}));
    }
    {   // a * b.conj() and a.norm() / b
        Combine<Complex32, Complex32, Complex32> cm(inst, B2S_COMBINE_CONJ_MUL_C32);
        cm.in0.set({{1, 2}, {3, -4}});
        cm.in1.set({{5, 6}, {-7, 0.5f}});
        cm.output.reserve(2);
        run(cm);
        auto y = cm.output.get();
        CHECK(y.size() == 2 && y[0] == Complex32(1 * 5.f - 2 * -6.f, 1 * -6.f + 2 * 5.f) &&
              y[1] == Complex32(3 * -7.f - (-4) * -0.5f, 3 * -0.5f + (-4) * -7.f));
        Combine<Complex32, float, float> md(inst, B2S_COMBINE_MAG_DIV_C32_F32);
        md.in0.set({{3, 4}, {INFINITY, NAN}, {5, 12}});
        md.in1.set({2, 1, 13});
        md.output.reserve(3);
        run(md);
        auto z = md.output.get();
        CHECK(z.size() == 3 && z[0] == 2.5f && std::isinf(z[1]) && z[1] > 0 && z[2] == 1.0f);
    }
    {   // tests/split.rs:8-43
        Split<Complex32> s(inst, B2S_SPLIT_RE_IM);
        std::vector<Complex32> x;
        std::vector<float> re, im;
        for (int k = 0; k < 10; k++) { x.push_back(Complex32((float)k, (float)k + 1)); re.push_back((float)k); im.push_back((float)k + 1); }
        s.input.set(x);
        s.output0.reserve(10);
        s.output1.reserve(10);
        WorkIo io = run(s);
        CHECK(io.finished && s.output0.get() == re && s.output1.get() == im);
    }
    {   // Delay: pad 3 (the mocker's input reports finished, so the call that completes the pad finishes the block,
        // delay.rs:131-136); skip 2, copy; new_value
        Delay<float> d(inst, 3);
        d.input.set({1, 2, 3, 4});
        d.output.reserve(10);
        WorkIo io = run(d);
        CHECK(io.finished && d.output.get() == std::vector<float>({0, 0, 0}) && d.state() == Delay<float>::State::Copy);
        Delay<float> s(inst, -2);
        s.input.set({1, 2, 3, 4});
        s.output.reserve(10);
        io = run(s);
        CHECK(io.finished && s.output.get() == std::vector<float>({3, 4}));
        s.new_value(true, 4);
        CHECK(s.state() == Delay<float>::State::Pad && s.count() == 4);
        s.new_value(false, 6);
        CHECK(s.state() == Delay<float>::State::Skip && s.count() == 2);
    }
    {   // StreamDuplicator<f64, 3> and StreamDeinterleaver<Complex32>(3)
        StreamDuplicator<double> dup(inst, 3);
        std::vector<double> x = {1.5, -2.25, 1e300, 5e-324, -0.0};
        dup.input.set(x);
        for (int k = 0; k < 3; k++) dup.out(k).reserve(8);
        WorkIo io = run(dup);
        CHECK(io.finished);
        for (int k = 0; k < 3; k++) {
            auto y = dup.out(k).get();
            CHECK(y.size() == x.size() && std::memcmp(y.data(), x.data(), x.size() * sizeof(double)) == 0);
        }
        StreamDeinterleaver<Complex32> de(inst, 3);
        std::vector<Complex32> v;
        for (int k = 0; k < 11; k++) v.push_back(Complex32((float)k, -(float)k));
        de.input.set(v);
        for (int k = 0; k < 3; k++) de.out(k).reserve(8);
        io = run(de);
        CHECK(io.finished);                                     // 2 items left < N (stream_deinterleaver.rs:91-95)
        for (int k = 0; k < 3; k++) {
            auto y = de.out(k).get();
            CHECK(y.size() == 3 && y[0] == v[k] && y[1] == v[3 + k] && y[2] == v[6 + k]);
        }
        bool refused = false;
        try { StreamDuplicator<float> big(inst, 257); } catch (const Error &e) { refused = e.code == B2S_EUNSUPPORTED; }
        CHECK(refused);
    }
    {   // firdes/basic.rs:229-247 and the SSB graph's taps
        auto t = firdes::hilbert(std::vector<double>(11, 1.0));
        CHECK(t.size() == 11 && t[1] == 0 && t[3] == 0 && t[5] == 0 && t[7] == 0 && t[9] == 0);
        CHECK(std::fabs(t[0]) == std::fabs(t[10]) && std::fabs(t[2]) == std::fabs(t[8]) && std::fabs(t[4]) == std::fabs(t[6]));
        CHECK(t[0] > t[2] && t[2] > t[4] && t[6] > t[8] && t[8] > t[10]);
        auto w = windows::hamming(38, false);
        CHECK(w.size() == 38 && std::fabs(w[1] - 0.086616681240054) < 1e-5 && std::fabs(w[18] - 0.998342844729562) < 1e-5);
        CHECK(firdes::hilbert(windows::hamming(167, false)).size() == 167);
        bool refused = false;
        try { firdes::hilbert(std::vector<double>(10, 1.0)); } catch (const Error &e) { refused = e.code == B2S_EINVAL; }
        CHECK(refused);
    }
    inst.sync();
    CHECK(b2s_ctx_bytes_held(inst.get()) == held);
    return report();
}
