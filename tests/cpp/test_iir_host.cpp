// test_iir_host.cpp -- the reference's IirFilter tests (crates/futuredsp/src/iir.rs:23-31, :186-236) replayed through
// the C++ host layer (include/b200sdr.hpp) on a GPU, under every algorithm that admits the filter.
// Built by __graft_entry__.build(); run by tests/test_gpu_cpp_host.py (needs an H100).
#include <cstdio>
#include <optional>

#include "b200sdr.hpp"
#include "check.hpp"

using namespace b2s;

// the Feeder of iir.rs:186-203: append one sample, filter into a one-item slice, drain what was consumed
struct Feeder {
    IirFilter<float> &filter;
    std::vector<float> input;
    std::optional<float> feed(float v) {
        input.push_back(v);
        std::vector<float> out(1, 0.f);
        auto [c, p, st] = filter.filter(input, out);
        (void)st;
        CHECK(c == p);
        input.erase(input.begin(), input.begin() + (long)c);
        if (p) return out[0];
        return std::nullopt;
    }
};

int main() {
    Instance inst(0);
    for (b2s_algo algo : {B2S_ALGO_AUTO, B2S_ALGO_DIRECT}) {
        {   // iir.rs:218-226 test_iir_b_taps_algorithm
            IirFilter<float> f(inst, {}, {1.0f, 2.0f, 3.0f}, algo);
            CHECK(f.length() == 3);
            Feeder fd{f, {}};
            CHECK(!fd.feed(10.0f));
            CHECK(!fd.feed(20.0f));
            CHECK(fd.feed(30.0f) == std::optional<float>(30.0f + 40.0f + 30.0f));
            CHECK(fd.feed(40.0f) == std::optional<float>(40.0f + 60.0f + 60.0f));
        }
        {   // iir.rs:23-31 doc example
            IirFilter<float> f(inst, {1.0f, 2.0f, 3.0f}, {4.0f, 5.0f, 6.0f}, algo);
            std::vector<float> in{1, 2, 3, 4, 5}, out(1, 0.f);
            f.filter(in, out);
            CHECK(out[0] == 42.0f);
        }
    }
    for (b2s_algo algo : {B2S_ALGO_AUTO, B2S_ALGO_DIRECT, B2S_ALGO_SCAN}) {   // iir.rs:228-236 test_iir_single_a_tap_algorithm
        IirFilter<float> f(inst, {0.5f}, {1.0f}, algo);
        CHECK(f.algo() == (algo == B2S_ALGO_DIRECT ? B2S_ALGO_DIRECT : B2S_ALGO_SCAN));
        Feeder fd{f, {}};
        CHECK(!fd.feed(10.0f));
        CHECK(fd.feed(10.0f) == std::optional<float>(15.0f));
        CHECK(fd.feed(10.0f) == std::optional<float>(17.5f));
        CHECK(fd.feed(10.0f) == std::optional<float>(18.75f));
    }
    {   // f64 impl (iir.rs:67-76): same vector, and SCAN is refused
        IirFilter<double> f(inst, {0.5}, {1.0});
        CHECK(f.algo() == B2S_ALGO_DIRECT);
        bool refused = false;
        try { f.set_algo(B2S_ALGO_SCAN); } catch (const Error &e) { refused = e.code == B2S_EUNSUPPORTED; }
        CHECK(refused);
        std::vector<double> in1{10}, in{10, 10, 10, 10}, out(4, 0.0);
        CHECK(std::get<1>(f.filter(in1, out)) == 0);            // fills memory only (:119-129)
        auto r = f.filter(in, out);
        CHECK(std::get<0>(r) == 4 && std::get<1>(r) == 4);
        CHECK(out[0] == 15.0 && out[1] == 17.5 && out[2] == 18.75 && out[3] == 19.375);
    }
    {   // n_b == 0: the reference asserts (:132)
        bool refused = false;
        try { IirFilter<float> f(inst, {0.5f}, {}); } catch (const Error &e) { refused = e.code == B2S_EINVAL; }
        CHECK(refused);
    }
    {   // blocks::Iir under Mocker (src/blocks/iir.rs:156-175)
        auto blk = IirBuilder::same_type<float>(inst, {0.5f}, {1.0f});
        CHECK(blk.length() == 1);
        Mocker<Iir<float>> m(blk);
        m.input(std::vector<float>{10, 10, 10, 10});
        m.init_output(8);
        m.run();                                                  // fills memory from x[0], then 4 outputs
        auto y = m.output();
        CHECK(y.size() == 4 && y[0] == 15.0f && y[1] == 17.5f && y[2] == 18.75f && y[3] == 19.375f);
    }
    inst.sync();
    return report();
}
