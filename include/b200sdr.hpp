// b200sdr.hpp -- C++ host layer above the C ABI (include/b200sdr.h), mirroring the reference's
// Rust interfaces for the hot path so call sites and tests read like the reference's own:
//
//   futuredsp::Filter::filter(&self, &[In], &mut [Out]) -> (usize, usize, ComputationStatus)
//                                     (crates/futuredsp/src/lib.rs:48-68)
//   futuredsp::{FirFilter, DecimatingFirFilter, PolyphaseResamplingFir, IirFilter}
//   futuresdr::blocks::{Fir, FirBuilder, Iir, IirBuilder, Fft, Apply, PfbArbResampler, SignalSource,
//                       SignalSourceBuilder, FixedPointPhase, Head, Combine, Split, Delay,
//                       StreamDuplicator, StreamDeinterleaver}                          (src/blocks/*.rs)
//   futuredsp::{firdes::{hilbert, lowpass}, windows::hamming}
//   futuresdr::runtime::{WorkIo, mocker::Mocker}                        (work_io.rs, mocker.rs)
//
// The reference is Rust; no Rust toolchain exists in this image, so this header is the
// compiled-language host side (INTEGRATION.md carries the Rust shim source).  Header-only,
// C++17, links against libb200sdr.so.  Errors the reference panics/asserts on throw b2s::Error.
#pragma once

#include <algorithm>
#include <array>
#include <complex>
#include <cstdint>
#include <cstring>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include "b200sdr.h"

namespace b2s {

using Complex32 = std::complex<float>;

struct Error : std::runtime_error {
    int32_t code;
    Error(int32_t c, const std::string &m) : std::runtime_error(m), code(c) {}
};

inline void check(int32_t rc, const b2s_ctx *ctx = nullptr) {
    if (rc < 0) throw Error(rc, std::string("libb200sdr: ") + b2s_last_error(ctx));
}

// Owner of one ABI object: destroyed with its b2s_*_destroy when the owner goes away, so an owner is move-only and a
// constructor that throws after the create call still frees what it created.
template <typename T, void (*Destroy)(T *)> struct HandleDeleter { void operator()(T *p) const { Destroy(p); } };
template <typename T, void (*Destroy)(T *)> using Handle = std::unique_ptr<T, HandleDeleter<T, Destroy>>;
// The out-parameter of a create call, handed to the Handle at the end of the full expression:
//     check(b2s_fft_plan_c32(..., out_ptr(plan_)), ...);
template <typename H> struct OutPtr {
    H &h;
    typename H::pointer p = nullptr;
    ~OutPtr() { h.reset(p); }
    operator typename H::pointer *() { return &p; }
};
template <typename H> OutPtr<H> out_ptr(H &h) { return OutPtr<H>{h}; }

// futuredsp::ComputationStatus (lib.rs:33-45)
enum class ComputationStatus : int32_t { InsufficientInput = 0, InsufficientOutput = 1, BothSufficient = 2 };
using FilterResult = std::tuple<size_t, size_t, ComputationStatus>;

// ≙ runtime::buffer::vulkan::Instance (buffer/vulkan/mod.rs:45-153)
class Instance {
public:
    explicit Instance(int device = 0) { check(b2s_ctx_create(device, out_ptr(ctx_))); }
    b2s_ctx *get() const { return ctx_.get(); }
    void sync() const { check(b2s_ctx_sync(ctx_.get()), ctx_.get()); }
    uint64_t launch_count() const { return b2s_ctx_launch_count(ctx_.get()); }

    template <typename T> T *device_alloc(size_t items) const {
        void *p = nullptr;
        check(b2s_malloc(ctx_.get(), items * sizeof(T), &p), ctx_.get());
        return static_cast<T *>(p);
    }
    void device_free(void *p) const { b2s_free(ctx_.get(), p); }
    template <typename T> void upload(T *dst, const T *src, size_t items) const {
        check(b2s_memcpy_h2d(ctx_.get(), dst, src, items * sizeof(T)), ctx_.get());
    }
    template <typename T> void download(T *dst, const T *src, size_t items) const {
        check(b2s_memcpy_d2h(ctx_.get(), dst, src, items * sizeof(T)), ctx_.get());
        sync();
    }

private:
    Handle<b2s_ctx, b2s_ctx_destroy> ctx_;
};

template <typename Sample, typename Tap> constexpr b2s_kind kind_of() {
    if constexpr (std::is_same_v<Sample, float> && std::is_same_v<Tap, float>) return B2S_F32_F32;
    else if constexpr (std::is_same_v<Sample, Complex32> && std::is_same_v<Tap, float>) return B2S_C32_F32;
    else {
        static_assert(std::is_same_v<Sample, Complex32> && std::is_same_v<Tap, Complex32>,
                      "no futuredsp impl for this sample/tap combination");
        return B2S_C32_C32;
    }
}

// ---- futuredsp::Filter ----------------------------------------------------------------------
template <typename Sample> class Filter {
public:
    virtual ~Filter() = default;
    // host slices (Filter::filter(&[In], &mut [Out]))
    virtual FilterResult filter(const Sample *input, size_t n_in, Sample *output, size_t n_out) const = 0;
    // device slices (samples already in HBM; asynchronous on the instance's stream)
    virtual FilterResult filter_device(const Sample *d_in, size_t n_in, Sample *d_out, size_t n_out) const = 0;
    virtual size_t length() const = 0;
    FilterResult filter(const std::vector<Sample> &i, std::vector<Sample> &o) const {
        return filter(i.data(), i.size(), o.data(), o.size());
    }
};

// ≙ DecimatingFirFilter (decimating_fir.rs:31-95); decimation 1 == FirFilter (fir.rs:31-91)
template <typename Sample, typename Tap> class DecimatingFirFilter : public Filter<Sample> {
public:
    DecimatingFirFilter(const Instance &inst, size_t decimation, const std::vector<Tap> &taps, b2s_algo algo = B2S_ALGO_AUTO)
        : inst_(inst) {
        check(b2s_fir_plan(inst.get(), kind_of<Sample, Tap>(), reinterpret_cast<const float *>(taps.data()), taps.size(),
                           decimation, out_ptr(plan_)), inst.get());
        if (algo != B2S_ALGO_AUTO) check(b2s_fir_set_algo(plan_.get(), algo), inst.get());
    }
    FilterResult filter(const Sample *i, size_t n_in, Sample *o, size_t n_out) const override {
        size_t c = 0, p = 0; int32_t st = 0;
        check(b2s_fir_filter_host(plan_.get(), i, n_in, o, n_out, &c, &p, &st), inst_.get());
        return {c, p, static_cast<ComputationStatus>(st)};
    }
    FilterResult filter_device(const Sample *i, size_t n_in, Sample *o, size_t n_out) const override {
        size_t c = 0, p = 0; int32_t st = 0;
        check(b2s_fir_exec(plan_.get(), i, n_in, o, n_out, &c, &p, &st), inst_.get());
        return {c, p, static_cast<ComputationStatus>(st)};
    }
    using Filter<Sample>::filter;
    size_t length() const override { return b2s_fir_length(plan_.get()); }
    int algo() const { return b2s_fir_get_algo(plan_.get()); }

protected:
    const Instance &inst_;
    Handle<b2s_fir, b2s_fir_destroy> plan_;
};

template <typename Sample, typename Tap> class FirFilter : public DecimatingFirFilter<Sample, Tap> {
public:
    FirFilter(const Instance &inst, const std::vector<Tap> &taps, b2s_algo algo = B2S_ALGO_AUTO)
        : DecimatingFirFilter<Sample, Tap>(inst, 1, taps, algo) {}
};

// ≙ PolyphaseResamplingFir (polyphase_resampling_fir.rs:42-124); device slices only
template <typename Sample> class PolyphaseResamplingFir : public Filter<Sample> {
public:
    PolyphaseResamplingFir(const Instance &inst, size_t interp, size_t decim, const std::vector<float> &taps)
        : inst_(inst) {
        check(b2s_resamp_plan(inst.get(), kind_of<Sample, float>(), taps.data(), taps.size(), interp, decim, out_ptr(plan_)),
              inst.get());
    }
    FilterResult filter(const Sample *i, size_t n_in, Sample *o, size_t n_out) const override {
        // host slices: stage through device memory (no internal pipeline for this core yet)
        Sample *di = inst_.device_alloc<Sample>(n_in + 1), *dout = inst_.device_alloc<Sample>(n_out + 1);
        inst_.upload(di, i, n_in);
        auto r = filter_device(di, n_in, dout, n_out);
        inst_.download(o, dout, std::get<1>(r));
        inst_.device_free(di); inst_.device_free(dout);
        return r;
    }
    FilterResult filter_device(const Sample *i, size_t n_in, Sample *o, size_t n_out) const override {
        size_t c = 0, p = 0; int32_t st = 0;
        check(b2s_resamp_exec(plan_.get(), i, n_in, o, n_out, &c, &p, &st), inst_.get());
        return {c, p, static_cast<ComputationStatus>(st)};
    }
    using Filter<Sample>::filter;
    size_t length() const override { return b2s_resamp_length(plan_.get()); }

private:
    const Instance &inst_;
    Handle<b2s_resamp, b2s_resamp_destroy> plan_;
};

// ≙ futuredsp::IirFilter (crates/futuredsp/src/iir.rs:33-178), a StatefulFilter: memory and its fill count live in the
// plan, so filter() is non-const and consecutive calls continue one stream.  Sample = float or double (:56-76).
template <typename Sample> class IirFilter {
    static_assert(std::is_same_v<Sample, float> || std::is_same_v<Sample, double>, "IirFilter: f32 or f64 only");
public:
    IirFilter(const Instance &inst, const std::vector<Sample> &a_taps, const std::vector<Sample> &b_taps,
              b2s_algo algo = B2S_ALGO_AUTO)
        : inst_(inst) {
        if constexpr (std::is_same_v<Sample, float>)
            check(b2s_iir_plan_f32(inst.get(), a_taps.data(), a_taps.size(), b_taps.data(), b_taps.size(), out_ptr(plan_)), inst.get());
        else
            check(b2s_iir_plan_f64(inst.get(), a_taps.data(), a_taps.size(), b_taps.data(), b_taps.size(), out_ptr(plan_)), inst.get());
        if (algo != B2S_ALGO_AUTO) set_algo(algo);
    }
    void set_algo(b2s_algo algo) { check(b2s_iir_set_algo(plan_.get(), algo), inst_.get()); }
    int algo() const { return b2s_iir_get_algo(plan_.get()); }
    size_t length() const { return b2s_iir_length(plan_.get()); }
    // device slices (asynchronous on the instance's stream)
    FilterResult filter_device(const Sample *i, size_t n_in, Sample *o, size_t n_out) {
        size_t c = 0, p = 0; int32_t st = 0;
        check(b2s_iir_exec(plan_.get(), i, n_in, o, n_out, &c, &p, &st), inst_.get());
        return {c, p, static_cast<ComputationStatus>(st)};
    }
    // host slices: staged through device memory
    FilterResult filter(const Sample *i, size_t n_in, Sample *o, size_t n_out) {
        Sample *di = inst_.device_alloc<Sample>(n_in + 1), *dout = inst_.device_alloc<Sample>(n_out + 1);
        inst_.upload(di, i, n_in);
        auto r = filter_device(di, n_in, dout, n_out);
        inst_.download(o, dout, std::get<1>(r));
        inst_.device_free(di); inst_.device_free(dout);
        return r;
    }
    FilterResult filter(const std::vector<Sample> &i, std::vector<Sample> &o) { return filter(i.data(), i.size(), o.data(), o.size()); }

private:
    const Instance &inst_;
    Handle<b2s_iir, b2s_iir_destroy> plan_;
};

// ---- firdes (futuredsp::firdes::kaiser, firdes/basic.rs:310-459) ---------------------------------
namespace firdes::kaiser {
inline std::vector<float> lowpass(double cutoff, double transition_bw, double max_ripple) {
    std::vector<float> t(b2s_firdes_kaiser_lowpass(cutoff, transition_bw, max_ripple, nullptr, 0));
    if (t.empty()) throw Error(B2S_EINVAL, "firdes::kaiser::lowpass: bad specification");
    b2s_firdes_kaiser_lowpass(cutoff, transition_bw, max_ripple, t.data(), t.size());
    return t;
}
inline std::vector<float> multirate(size_t interp, size_t decim, size_t half_len, double max_ripple) {
    std::vector<float> t(b2s_firdes_kaiser_multirate(interp, decim, half_len, max_ripple, nullptr, 0));
    if (t.empty()) throw Error(B2S_EINVAL, "firdes::kaiser::multirate: bad specification");
    b2s_firdes_kaiser_multirate(interp, decim, half_len, max_ripple, t.data(), t.size());
    return t;
}
}  // namespace firdes::kaiser

// ---- runtime pieces the blocks need -----------------------------------------------------------
struct WorkIo { bool call_again = false, finished = false; };   // work_io.rs:11-34

// mocker::Reader / mocker::Writer (mocker.rs:213-400) over device memory
template <typename T> class Reader {
public:
    explicit Reader(const Instance &i) : inst_(i) {}
    ~Reader() { if (d_) inst_.device_free(d_); }
    Reader(const Reader &) = delete;
    Reader &operator=(const Reader &) = delete;
    void set(const std::vector<T> &v) {
        if (d_) inst_.device_free(d_);
        d_ = inst_.device_alloc<T>(v.size() + 1); n_ = v.size(); pos_ = 0;
        inst_.upload(d_, v.data(), v.size());
    }
    const T *slice() const { return d_ + pos_; }
    size_t len() const { return n_ - pos_; }
    void consume(size_t n) { pos_ += n; }
    bool finished() const { return true; }
private:
    const Instance &inst_; T *d_ = nullptr; size_t n_ = 0, pos_ = 0;
};
template <typename T> class Writer {
public:
    explicit Writer(const Instance &i) : inst_(i) {}
    ~Writer() { if (d_) inst_.device_free(d_); }
    Writer(const Writer &) = delete;
    Writer &operator=(const Writer &) = delete;
    void reserve(size_t n) { if (d_) inst_.device_free(d_); d_ = inst_.device_alloc<T>(n + 1); cap_ = n; len_ = 0; }
    T *slice() { return d_ + len_; }
    size_t capacity() const { return cap_ - len_; }
    void produce(size_t n) { len_ += n; }
    std::vector<T> get() const { std::vector<T> v(len_); if (len_) inst_.download(v.data(), d_, len_); return v; }
private:
    const Instance &inst_; T *d_ = nullptr; size_t cap_ = 0, len_ = 0;
};

// ≙ blocks::Fir (src/blocks/fir.rs:13-95)
template <typename Sample> class Fir {
public:
    Fir(const Instance &inst, std::unique_ptr<Filter<Sample>> core) : input(inst), output(inst), filter_(std::move(core)) {}
    size_t n_taps() const { return filter_->length(); }
    void work(WorkIo &io) {                                                        // fir.rs:75-94
        auto [consumed, produced, status] = filter_->filter_device(input.slice(), input.len(), output.slice(), output.capacity());
        input.consume(consumed);
        output.produce(produced);
        if (input.finished() && status != ComputationStatus::InsufficientOutput) io.finished = true;
    }
    Reader<Sample> input;
    Writer<Sample> output;
private:
    std::unique_ptr<Filter<Sample>> filter_;
};

// ≙ blocks::FirBuilder (src/blocks/fir.rs:126-233)
struct FirBuilder {
    template <typename Sample, typename Tap>
    static Fir<Sample> fir(const Instance &i, const std::vector<Tap> &taps) {
        return Fir<Sample>(i, std::make_unique<FirFilter<Sample, Tap>>(i, taps));
    }
    template <typename Sample> static Fir<Sample> decimating(const Instance &i, size_t decim) {
        return decimating_with_taps<Sample, float>(i, decim, firdes::kaiser::lowpass(1.0 / (double)decim, 0.1, 0.0001));   // fir.rs:154
    }
    template <typename Sample, typename Tap>
    static Fir<Sample> decimating_with_taps(const Instance &i, size_t decim, const std::vector<Tap> &taps) {
        return Fir<Sample>(i, std::make_unique<DecimatingFirFilter<Sample, Tap>>(i, decim, taps));
    }
    template <typename Sample> static Fir<Sample> resampling(const Instance &i, size_t interp, size_t decim) {
        size_t a = interp, b = decim;
        while (b) { size_t t = a % b; a = b; b = t; }                               // gcd (fir.rs:197-199)
        interp /= a; decim /= a;
        return resampling_with_taps<Sample>(i, interp, decim, firdes::kaiser::multirate(interp, decim, 12, 0.0001));
    }
    template <typename Sample>
    static Fir<Sample> resampling_with_taps(const Instance &i, size_t interp, size_t decim, const std::vector<float> &taps) {
        if (taps.size() % interp) throw Error(B2S_EINVAL, "taps.num_taps().is_multiple_of(interp)");   // :56
        return Fir<Sample>(i, std::make_unique<PolyphaseResamplingFir<Sample>>(i, interp, decim, taps));
    }
};

// ≙ blocks::Iir (src/blocks/iir.rs:8-176)
template <typename Sample> class Iir {
public:
    Iir(const Instance &inst, std::unique_ptr<IirFilter<Sample>> core) : input(inst), output(inst), core_(std::move(core)) {}
    size_t length() const { return core_->length(); }                                  // set_min_items(n_b), :133
    void work(WorkIo &io) {                                                        // iir.rs:156-175
        auto [consumed, produced, status] = core_->filter_device(input.slice(), input.len(), output.slice(), output.capacity());
        input.consume(consumed);
        output.produce(produced);
        if (input.finished() && status != ComputationStatus::InsufficientOutput) io.finished = true;
    }
    Reader<Sample> input;
    Writer<Sample> output;
private:
    std::unique_ptr<IirFilter<Sample>> core_;
};

// ≙ blocks::IirBuilder (src/blocks/iir.rs:32-64)
struct IirBuilder {
    template <typename Sample>
    static Iir<Sample> iir(const Instance &i, const std::vector<Sample> &a_taps, const std::vector<Sample> &b_taps) {
        return Iir<Sample>(i, std::make_unique<IirFilter<Sample>>(i, a_taps, b_taps));
    }
    template <typename Sample>
    static Iir<Sample> same_type(const Instance &i, const std::vector<Sample> &a_taps, const std::vector<Sample> &b_taps) {
        return iir<Sample>(i, a_taps, b_taps);
    }
};

// ≙ blocks::FixedPointPhase (src/blocks/signal_source/fxpt_phase.rs:8-99), evaluated on the host by the library
struct FixedPointPhase {
    int32_t value = 0;
    static FixedPointPhase make(float x) { FixedPointPhase p; check(b2s_fxpt_phase_new(x, &p.value)); return p; }   // ::new
    float sin() const { float s, c; check(b2s_fxpt_sin_cos(value, &s, &c)); return s; }
    float cos() const { float s, c; check(b2s_fxpt_sin_cos(value, &s, &c)); return c; }
};

// ≙ blocks::SignalSource (src/blocks/signal_source/mod.rs:29-108): no input; work() fills the whole output slice and
// never finishes.  T = float or Complex32.
template <typename T> class SignalSource {
    static_assert(std::is_same_v<T, float> || std::is_same_v<T, Complex32>, "SignalSource: f32 or Complex32 items");
public:
    SignalSource(const Instance &inst, b2s_wave wave, float frequency, float sample_rate, float amplitude,
                 float initial_phase)
        : output(inst), inst_(inst) {
        check(b2s_sigsrc_create(inst.get(), wave, std::is_same_v<T, Complex32> ? 1 : 0, frequency, sample_rate,
                                amplitude, initial_phase, out_ptr(h_)), inst.get());
    }
    void set_amplitude(float amplitude) { check(b2s_sigsrc_set_amplitude(h_.get(), amplitude), inst_.get()); }   // :71-73
    // (the next sample's phase, the increment)
    std::pair<FixedPointPhase, FixedPointPhase> phase() const {
        FixedPointPhase v, inc;
        check(b2s_sigsrc_phase(h_.get(), &v.value, &inc.value), inst_.get());
        return {v, inc};
    }
    void work(WorkIo &) {                                                           // mod.rs:88-107
        size_t p = 0;
        check(b2s_sigsrc_exec(h_.get(), output.slice(), output.capacity(), &p), inst_.get());
        output.produce(p);
    }
    Writer<T> output;
private:
    const Instance &inst_; Handle<b2s_sigsrc, b2s_sigsrc_destroy> h_;
};

// ≙ blocks::SignalSourceBuilder (src/blocks/signal_source/mod.rs:110-227)
template <typename T> struct SignalSourceBuilder {
    static SignalSource<T> cos(const Instance &i, float frequency, float sample_rate, float amplitude, float initial_phase) {
        return SignalSource<T>(i, B2S_WAVE_COS, frequency, sample_rate, amplitude, initial_phase);
    }
    static SignalSource<T> sin(const Instance &i, float frequency, float sample_rate, float amplitude, float initial_phase) {
        return SignalSource<T>(i, B2S_WAVE_SIN, frequency, sample_rate, amplitude, initial_phase);
    }
    static SignalSource<T> square(const Instance &i, float frequency, float sample_rate, float amplitude, float initial_phase) {
        return SignalSource<T>(i, B2S_WAVE_SQUARE, frequency, sample_rate, amplitude, initial_phase);
    }
};

// ≙ blocks::Head (src/blocks/head.rs:22-84): copies the first n_items items, finishes when n_items reaches 0
template <typename T> class Head {
public:
    Head(const Instance &inst, uint64_t n_items) : input(inst), output(inst), inst_(inst), n_items_(n_items) {}
    uint64_t n_items() const { return n_items_; }
    void work(WorkIo &io) {                                                        // head.rs:57-83
        const size_t m = (size_t)std::min<uint64_t>(n_items_, std::min(input.len(), output.capacity()));
        if (m > 0) {
            check(b2s_memcpy_d2d(inst_.get(), output.slice(), input.slice(), m * sizeof(T)), inst_.get());
            n_items_ -= m;
            if (n_items_ == 0) io.finished = true;
            input.consume(m);
            output.produce(m);
        }
    }
    Reader<T> input;
    Writer<T> output;
private:
    const Instance &inst_; uint64_t n_items_;
};

// ≙ blocks::Fft (src/blocks/fft.rs:30-221)
enum class FftDirection { Forward, Inverse };
class Fft {
public:
    Fft(const Instance &inst, size_t len, FftDirection dir = FftDirection::Forward, bool fft_shift = false,
        bool has_normalize = false, float normalize = 1.0f)
        : input(inst), output(inst), inst_(inst), len_(len) {
        check(b2s_fft_plan_c32(inst.get(), len, dir == FftDirection::Inverse, fft_shift, has_normalize, normalize, out_ptr(plan_)), inst.get());
    }
    void work(WorkIo &io) {                                                        // fft.rs:160-221
        size_t c = 0, p = 0;
        check(b2s_fft_exec(plan_.get(), input.slice(), input.len(), output.slice(), output.capacity(), &c, &p), inst_.get());
        input.consume(c); output.produce(p);
        if (input.finished() && c == (c / len_) * len_) io.finished = true;
    }
    Reader<Complex32> input;
    Writer<Complex32> output;
private:
    const Instance &inst_; size_t len_; Handle<b2s_fft, b2s_fft_destroy> plan_;
};

// ≙ blocks::Apply (src/blocks/apply.rs:100-131) for the device op catalogue; B2S_OP_SLICE_F32_U8 is Apply<float, uint8_t>
template <typename A, typename B> class Apply {
public:
    Apply(const Instance &inst, b2s_op op, float param = 1.0f) : input(inst), output(inst), inst_(inst) {
        check(b2s_apply_create(inst.get(), op, param, out_ptr(h_)), inst.get());
    }
    void work(WorkIo &io) {
        const size_t i_len = input.len();
        size_t c = 0, p = 0;
        check(b2s_apply_exec(h_.get(), input.slice(), i_len, output.slice(), output.capacity(), &c, &p), inst_.get());
        input.consume(c); output.produce(p);
        if (input.finished() && c == i_len) io.finished = true;                     // apply.rs:126-128
    }
    Reader<A> input;
    Writer<B> output;
private:
    const Instance &inst_; Handle<b2s_apply, b2s_apply_destroy> h_;
};

// ≙ blocks::PfbArbResampler (src/blocks/pfb/arb_resampler.rs:72-231)
class PfbArbResampler {
public:
    PfbArbResampler(const Instance &inst, float rate, const std::vector<float> &taps, size_t num_filters)
        : input(inst), output(inst), inst_(inst) {
        check(b2s_pfbarb_plan_c32(inst.get(), taps.data(), taps.size(), num_filters, rate, out_ptr(h_)), inst.get());
    }
    void work(WorkIo &io) {
        size_t c = 0, p = 0; int32_t again = 0;
        const size_t n = input.len();
        check(b2s_pfbarb_exec(h_.get(), input.slice(), n, output.slice(), output.capacity(), &c, &p, &again), inst_.get());
        input.consume(c); output.produce(p);
        if (again) io.call_again = true;
        else if (n - c == 0 && input.finished()) io.finished = true;
    }
    Reader<Complex32> input;
    Writer<Complex32> output;
private:
    const Instance &inst_; Handle<b2s_pfbarb, b2s_pfbarb_destroy> h_;
};

// ≙ futuredsp::Rotator (crates/futuredsp/src/rotator.rs:13-48): phase recurrence replayed bit for bit
class Rotator {
public:
    Rotator(const Instance &inst, float phase_incr) : inst_(inst) { check(b2s_rotator_create(inst.get(), phase_incr, out_ptr(h_)), inst.get()); }
    // Rotator::rotate (:32-47) on device slices; d_in == d_out is rotate_inplace (:24-29)
    std::pair<size_t, ComputationStatus> rotate_device(const Complex32 *d_in, size_t n_in, Complex32 *d_out, size_t n_out) {
        size_t n = 0; int32_t st = 0;
        check(b2s_rotator_exec(h_.get(), d_in, n_in, d_out, n_out, &n, &st), inst_.get());
        return {n, static_cast<ComputationStatus>(st)};
    }
    void reset() { check(b2s_rotator_reset(h_.get()), inst_.get()); }
private:
    const Instance &inst_; Handle<b2s_rotator, b2s_rotator_destroy> h_;
};

// ≙ Apply over one of the SSB example's oscillator closures (b2s_mix_op): `osc *= shift; f(v, osc)`, bit for bit.
// Mixer<float> is the Weaver demodulator (c32 -> f32), Mixer<Complex32> the two ROTATE ops.
template <typename Out> class Mixer {
public:
    Mixer(const Instance &inst, b2s_mix_op op, float phase_incr, float param = 1.0f) : input(inst), output(inst), inst_(inst) {
        if ((op == B2S_MIX_WEAVER_F32) != std::is_same<Out, float>::value)
            throw Error(B2S_EINVAL, "Mixer: the Weaver op writes float, the ROTATE ops Complex32");
        check(b2s_mixer_create(inst.get(), op, phase_incr, param, out_ptr(h_)), inst.get());
    }
    // one exec on device slices -> (consumed, produced); d_in == d_out runs a ROTATE op in place
    std::pair<size_t, size_t> mix_device(const Complex32 *d_in, size_t n_in, Out *d_out, size_t n_out) {
        size_t c = 0, p = 0;
        check(b2s_mixer_exec(h_.get(), d_in, n_in, d_out, n_out, &c, &p), inst_.get());
        return {c, p};
    }
    void reset() { check(b2s_mixer_reset(h_.get()), inst_.get()); }
    void work(WorkIo &io) {                                                        // apply.rs:100-131
        const size_t i_len = input.len();
        auto [c, p] = mix_device(input.slice(), i_len, output.slice(), output.capacity());
        input.consume(c); output.produce(p);
        if (input.finished() && c == i_len) io.finished = true;
    }
    Reader<Complex32> input;
    Writer<Out> output;
private:
    const Instance &inst_; Handle<b2s_mixer, b2s_mixer_destroy> h_;
};

// ≙ blocks::XlatingFir (src/blocks/xlating_fir.rs:22-126): band-pass complex taps (:80-86), decimating FIR,
// Rotator at the output rate (:97-99, :118)
class XlatingFir {
public:
    XlatingFir(const Instance &inst, size_t decimation, float offset, float sample_rate)          // XlatingFir::new (:42-48)
        : XlatingFir(inst, default_taps(decimation), decimation, offset, sample_rate) {}
    XlatingFir(const Instance &inst, const std::vector<float> &taps, size_t decimation, float offset, float sample_rate)
        : input(inst), output(inst), inst_(inst) {
        if (decimation == 0) throw Error(B2S_EINVAL, "Xlating FIR: decimation must be > 0");
        std::vector<Complex32> bpf(taps.size());
        float incr = 0.f;
        check(b2s_xlating_taps(taps.data(), taps.size(), offset, sample_rate, decimation,
                               reinterpret_cast<float *>(bpf.data()), &incr));
        filter_ = std::make_unique<DecimatingFirFilter<Complex32, Complex32>>(inst, decimation, bpf);
        rotator_ = std::make_unique<Rotator>(inst, incr);
    }
    size_t n_taps() const { return filter_->length(); }
    void work(WorkIo &io) {                                                        // xlating_fir.rs:105-126
        auto [consumed, produced, status] = filter_->filter_device(input.slice(), input.len(), output.slice(), output.capacity());
        if (produced) rotator_->rotate_device(output.slice(), produced, output.slice(), produced);
        input.consume(consumed);
        output.produce(produced);
        if (input.finished() && status != ComputationStatus::InsufficientOutput) io.finished = true;
    }
    Reader<Complex32> input;
    Writer<Complex32> output;
private:
    static std::vector<float> default_taps(size_t decimation) {
        if (decimation < 2) throw Error(B2S_EINVAL, "Xlating FIR: Decimation has to be >= 2");   // :43
        const double transition_bw = 0.1;
        const double cutoff = std::min(0.5 - transition_bw - 2.220446049250313e-16, 1.0 / (double)decimation);
        return firdes::kaiser::lowpass(cutoff, transition_bw, 0.0001);
    }
    const Instance &inst_;
    std::unique_ptr<DecimatingFirFilter<Complex32, Complex32>> filter_;
    std::unique_ptr<Rotator> rotator_;
};

// ≙ blocks::MovingAvg<WIDTH> (src/blocks/moving_avg.rs:24-116)
class MovingAvg {
public:
    MovingAvg(const Instance &inst, size_t width, float decay_factor, size_t history_size)
        : input(inst), output(inst), inst_(inst), width_(width) {
        check(b2s_mavg_create(inst.get(), width, decay_factor, history_size, out_ptr(h_)), inst.get());   // asserts of :58-61 -> EINVAL
    }
    void work(WorkIo &io) {                                                        // moving_avg.rs:72-115
        const size_t n = input.len();
        size_t c = 0, p = 0;
        check(b2s_mavg_exec(h_.get(), input.slice(), n, output.slice(), output.capacity(), &c, &p), inst_.get());
        if (input.finished() && c / width_ == n / width_) io.finished = true;       // :106-108
        input.consume(c); output.produce(p);
    }
    Reader<float> input;
    Writer<float> output;
private:
    const Instance &inst_; size_t width_; Handle<b2s_mavg, b2s_mavg_destroy> h_;
};

// The spectrum flowgraph's compute chain as one block: Fft::with_options(n, Forward, fft_shift, None) ->
// Apply(norm_sqr) -> MovingAvg<n>::new(decay, history) of examples/spectrum/src/bin/cpu.rs:21-28 in ONE pass over the
// samples (b2s_spectrum_*); counts follow MovingAvg::work, values agree with the three blocks to rounding.
class SpectrumPipe {
public:
    SpectrumPipe(const Instance &inst, size_t n, float decay_factor, size_t history_size, bool fft_shift = true,
                 float log10_scale = 0.0f)
        : input(inst), output(inst), inst_(inst), n_(n) {
        check(b2s_spectrum_plan(inst.get(), n, fft_shift ? 1 : 0, decay_factor, history_size, log10_scale, out_ptr(h_)), inst.get());
    }
    void work(WorkIo &io) {
        const size_t n = input.len();
        size_t c = 0, p = 0;
        check(b2s_spectrum_exec(h_.get(), input.slice(), n, output.slice(), output.capacity(), &c, &p), inst_.get());
        if (input.finished() && c / n_ == n / n_) io.finished = true;               // moving_avg.rs:106-108
        input.consume(c); output.produce(p);
    }
    Reader<Complex32> input;
    Writer<float> output;
private:
    const Instance &inst_; size_t n_; Handle<b2s_spectrum, b2s_spectrum_destroy> h_;
};

// ---- stream plumbing of branching graphs (b2s_combine_exec / b2s_split_exec / b2s_fanout_exec) --------------------
// ≙ blocks::Combine (src/blocks/combine.rs:31-137) for the b2s_combine_op catalogue; A, B, Out are the op's item types
template <typename A, typename B, typename Out> class Combine {
public:
    Combine(const Instance &inst, b2s_combine_op op) : in0(inst), in1(inst), output(inst), inst_(inst), op_(op) {}
    void work(WorkIo &io) {                                                        // combine.rs:102-136
        const size_t i0_len = in0.len(), i1_len = in1.len();
        size_t c = 0, m = 0;
        check(b2s_combine_exec(inst_.get(), op_, in0.slice(), i0_len, in1.slice(), i1_len, output.slice(), output.capacity(),
                               &c, &m), inst_.get());
        if (m > 0) { in0.consume(m); in1.consume(m); output.produce(m); }
        if (in0.finished() && m == i0_len) io.finished = true;
        if (in1.finished() && m == i1_len) io.finished = true;
    }
    Reader<A> in0;
    Reader<B> in1;
    Writer<Out> output;
private:
    const Instance &inst_; b2s_combine_op op_;
};

// ≙ blocks::Split (src/blocks/split.rs:31-127): RE_IM (In = Complex32) or DUP_F32 (In = float), two f32 outputs
template <typename In> class Split {
public:
    Split(const Instance &inst, b2s_split_op op) : input(inst), output0(inst), output1(inst), inst_(inst), op_(op) {}
    void work(WorkIo &io) {                                                        // split.rs:95-126
        const size_t i_len = input.len();
        size_t c = 0, m = 0;
        check(b2s_split_exec(inst_.get(), op_, input.slice(), i_len, output0.slice(), output1.slice(),
                             std::min(output0.capacity(), output1.capacity()), &c, &m), inst_.get());
        if (m > 0) { input.consume(m); output0.produce(m); output1.produce(m); }
        if (input.finished() && m == i_len) io.finished = true;
    }
    Reader<In> input;
    Writer<float> output0, output1;
private:
    const Instance &inst_; b2s_split_op op_;
};

// ≙ blocks::Delay (src/blocks/delay.rs:31-169): n > 0 pads n zero items, n <= 0 skips -n items, then copies
template <typename T> class Delay {
public:
    enum class State { Pad, Skip, Copy };
    Delay(const Instance &inst, int64_t n) : input(inst), output(inst), inst_(inst) {
        if (n > 0) { state_ = State::Pad; n_ = (size_t)n; } else { state_ = State::Skip; n_ = (size_t)(-n); }
    }
    State state() const { return state_; }
    size_t count() const { return n_; }
    // the new_value message handler (delay.rs:68-105)
    void new_value(bool pad, size_t value) {
        const int64_t val = pad ? (int64_t)value : -(int64_t)value;
        const int64_t cur = state_ == State::Pad ? (int64_t)n_ : state_ == State::Skip ? -(int64_t)n_ : 0;
        const int64_t nv = cur + val;
        if (nv > 0) { state_ = State::Pad; n_ = (size_t)nv; }
        else if (nv == 0) { state_ = State::Copy; n_ = 0; }
        else { state_ = State::Skip; n_ = (size_t)(-nv); }
    }
    void work(WorkIo &io) {                                                        // delay.rs:114-168
        const size_t i_len = input.len(), o_len = output.capacity();
        if (state_ == State::Pad) {
            const size_t m = std::min(o_len, n_);
            if (m) check(b2s_memset(inst_.get(), output.slice(), 0, m * sizeof(T)), inst_.get());
            output.produce(m);
            if (m == n_) {
                state_ = State::Copy; n_ = 0;
                io.call_again = true;
                if (input.finished()) io.finished = true;
            } else n_ -= m;
        } else if (state_ == State::Skip) {
            const size_t m = std::min(i_len, n_);
            input.consume(m);
            if (m == n_) { state_ = State::Copy; n_ = 0; io.call_again = true; }
            else n_ -= m;
            if (input.finished() && m == i_len) io.finished = true;
        } else {
            const size_t m = std::min(i_len, o_len);
            if (m) check(b2s_memcpy_d2d(inst_.get(), output.slice(), input.slice(), m * sizeof(T)), inst_.get());
            input.consume(m);
            output.produce(m);
            if (input.finished() && m == i_len) io.finished = true;
        }
    }
    Reader<T> input;
    Writer<T> output;
private:
    const Instance &inst_; State state_; size_t n_ = 0;
};

// ≙ the WLAN and M17 receivers' MovingAverage (examples/wlan/src/moving_average.rs:27-107, T = float or Complex32;
// examples/m17/src/moving_average.rs:5-81, float with divisor 4800).  Not MovingAvg.  One work() runs the reference's
// work() calls back to back on the current slices until one makes no progress, or at most max_calls of them
// (1: exactly one reference call); call_again and the finish rule are those of the last call (b2s_boxavg_exec).
template <typename T> class MovingAverage {
    static_assert(std::is_same_v<T, float> || std::is_same_v<T, Complex32>, "MovingAverage: f32 or Complex32 items");
public:
    MovingAverage(const Instance &inst, size_t len, std::optional<float> divisor = std::nullopt, size_t max_calls = 0)
        : input(inst), output(inst), inst_(inst), max_calls_(max_calls) {
        check(b2s_boxavg_create(inst.get(), std::is_same_v<T, Complex32> ? 1 : 0, len, divisor.has_value(),
                                divisor.value_or(0.0f), out_ptr(h_)), inst.get());
    }
    void reset() { check(b2s_boxavg_reset(h_.get()), inst_.get()); }
    void work(WorkIo &io) {
        size_t c = 0, p = 0, calls = 0;
        int32_t again = 0, done = 0;
        check(b2s_boxavg_exec(h_.get(), input.slice(), input.len(), output.slice(), output.capacity(), max_calls_, &c,
                              &p, &calls, &again, &done), inst_.get());
        input.consume(c);
        output.produce(p);
        if (again) io.call_again = true;                                            // :82-84
        if (input.finished() && done) io.finished = true;                           // :103-105
    }
    Reader<T> input;
    Writer<T> output;
private:
    const Instance &inst_; size_t max_calls_; Handle<b2s_boxavg, b2s_boxavg_destroy> h_;
};

// Every record a b2s_*_drain_* function hands out for the block h, in stream order: it drains until a short read.
// Draining synchronises.
template <typename H, typename E>
std::vector<E> drain_records(int32_t (*fn)(H *, E *, size_t, size_t *), H *h, const b2s_ctx *ctx) {
    constexpr size_t chunk = 4096;
    std::vector<E> out;
    for (;;) {
        const size_t k = out.size();
        out.resize(k + chunk);
        size_t n = 0;
        check(fn(h, out.data() + k, chunk, &n), ctx);
        out.resize(k + n);
        if (n < chunk) return out;
    }
}

// ≙ the ADS-B receiver's PreambleDetector -> Demodulator -> Decoder::check_crc (examples/adsb/src/preamble_detector.rs
// :65-146, demodulator.rs:49-113, decoder.rs:57-73) as one block (b2s_adsb_*).  Three f32 stream inputs, no stream
// output; the detector's tags and the demodulated frames are drained from the block.  work() runs one exec and
// finishes once an input is finished and the scan has reached the limit set by the smallest finished input.
class AdsbDemod {
public:
    AdsbDemod(const Instance &inst, float threshold = 10.0f, bool forward_failed_crc = false)
        : in_samples(inst), in_nf(inst), in_preamble_cor(inst), inst_(inst) {
        check(b2s_adsb_create(inst.get(), threshold, forward_failed_crc ? 1 : 0, out_ptr(h_)), inst.get());
    }
    void reset() { check(b2s_adsb_reset(h_.get()), inst_.get()); }
    // one exec over device slices (asynchronous): (consumed from each input, done)
    std::pair<size_t, bool> exec(const float *s, size_t n_s, const float *nf, size_t n_nf, const float *corr,
                                 size_t n_corr, bool finished) {
        size_t c = 0;
        int32_t done = 0;
        check(b2s_adsb_exec(h_.get(), s, n_s, nf, n_nf, corr, n_corr, finished ? 1 : 0, &c, &done), inst_.get());
        return {c, done != 0};
    }
    void work(WorkIo &io) {
        const size_t n = std::min({in_samples.len(), in_nf.len(), in_preamble_cor.len()});
        // every mocker::Reader is finished: the final exec runs on the common length
        auto [c, done] = exec(in_samples.slice(), n, in_nf.slice(), n, in_preamble_cor.slice(), n, true);
        in_samples.consume(c);
        in_nf.consume(c);
        in_preamble_cor.consume(c);
        if (done) io.finished = true;
    }
    // every packet / detection since the last drain, in stream order (synchronises)
    std::vector<b2s_adsb_packet> drain_packets() { return drain_records(b2s_adsb_drain_packets, h_.get(), inst_.get()); }
    std::vector<b2s_adsb_detection> drain_detections() {
        return drain_records(b2s_adsb_drain_detections, h_.get(), inst_.get());
    }
    Reader<float> in_samples, in_nf, in_preamble_cor;
private:
    const Instance &inst_; Handle<b2s_adsb, b2s_adsb_destroy> h_;
};

// ≙ the ZigBee receiver's ClockRecoveryMm (examples/zigbee/src/clock_recovery_mm.rs:28-97), f32 -> f32 (b2s_mmclock_*).
// exec() synchronises once (consumption depends on the data); a step that would move past the slice (B2S_ESTATE)
// throws Error, with the block left before that step.  work() finishes once the input is finished and what is left of
// it is within the look-ahead, or the call consumed nothing while it produced (a latched mu).  The reference finishes as
// soon as its input is finished; here a finished input can still hold items, and those are processed first.
class ClockRecoveryMm {
public:
    ClockRecoveryMm(const Instance &inst, float omega, float gain_omega, float mu, float gain_mu,
                    float omega_relative_limit)
        : input(inst), output(inst), inst_(inst) {
        check(b2s_mmclock_create(inst.get(), omega, gain_omega, mu, gain_mu, omega_relative_limit, out_ptr(h_)),
              inst.get());
    }
    void reset() { check(b2s_mmclock_reset(h_.get()), inst_.get()); }
    size_t look_ahead() const { return b2s_mmclock_look_ahead(h_.get()); }
    // one call of the reference's loop over device slices: (consumed, produced)
    std::pair<size_t, size_t> exec(const float *in, size_t n_in, float *out, size_t n_out_cap) {
        size_t c = 0, p = 0;
        check(b2s_mmclock_exec(h_.get(), in, n_in, out, n_out_cap, &c, &p), inst_.get());
        return {c, p};
    }
    void work(WorkIo &io) {
        const size_t n = input.len();
        auto [c, p] = exec(input.slice(), n, output.slice(), output.capacity());
        input.consume(c);
        output.produce(p);
        if (input.finished() && (n - c <= look_ahead() || (c == 0 && p > 0))) io.finished = true;
    }
    Reader<float> input;
    Writer<float> output;
private:
    const Instance &inst_; Handle<b2s_mmclock, b2s_mmclock_destroy> h_;
};

// ≙ the ZigBee receiver's Decoder (examples/zigbee/src/decoder.rs:78-183) with Mac::check_crc (mac.rs:62-85)
// (b2s_zigbee_*).  One f32 stream input, no stream output; the frames the reference posts are drained from the block.
// Every exec consumes its whole slice and never synchronises; work() finishes when the input is finished (:174-176).
class ZigbeeDecoder {
public:
    ZigbeeDecoder(const Instance &inst, uint32_t threshold = 6) : input(inst), inst_(inst) {
        check(b2s_zigbee_create(inst.get(), threshold, out_ptr(h_)), inst.get());
    }
    void reset() { check(b2s_zigbee_reset(h_.get()), inst_.get()); }
    size_t exec(const float *in, size_t n_in) {
        size_t c = 0;
        check(b2s_zigbee_exec(h_.get(), in, n_in, &c), inst_.get());
        return c;
    }
    void work(WorkIo &io) {
        input.consume(exec(input.slice(), input.len()));
        if (input.finished()) io.finished = true;
    }
    // every frame since the last drain, in stream order (synchronises)
    std::vector<b2s_zigbee_frame> drain_frames() { return drain_records(b2s_zigbee_drain_frames, h_.get(), inst_.get()); }
    Reader<float> input;
private:
    const Instance &inst_; Handle<b2s_zigbee, b2s_zigbee_destroy> h_;
};

// ≙ the keyfob receiver's Decoder (examples/keyfob/src/decoder.rs:64-127 with print, :36-52) (b2s_keyfob_*).  One u8
// stream input, no stream output; the strings the reference logs are drained from the block as codes.  Every exec
// consumes its whole slice and never synchronises; work() finishes when the input is finished (:120-122).
class KeyfobDecoder {
public:
    explicit KeyfobDecoder(const Instance &inst) : input(inst), inst_(inst) {
        check(b2s_keyfob_create(inst.get(), out_ptr(h_)), inst.get());
    }
    void reset() { check(b2s_keyfob_reset(h_.get()), inst_.get()); }
    size_t exec(const uint8_t *in, size_t n_in) {
        size_t c = 0;
        check(b2s_keyfob_exec(h_.get(), in, n_in, &c), inst_.get());
        return c;
    }
    void work(WorkIo &io) {
        input.consume(exec(input.slice(), input.len()));
        if (input.finished()) io.finished = true;
    }
    // every code since the last drain, in stream order (synchronises)
    std::vector<b2s_keyfob_code> drain_codes() { return drain_records(b2s_keyfob_drain_codes, h_.get(), inst_.get()); }
    Reader<uint8_t> input;
private:
    const Instance &inst_; Handle<b2s_keyfob, b2s_keyfob_destroy> h_;
};

// ≙ examples/lora/src/encoder.rs:33-284 over a batch: frame i is lengths[i] bytes of d_payloads (device, back to
// back); its symbols follow frame i - 1's in d_symbols.  Returns the symbol total.
inline size_t lora_encode(const Instance &inst, int sf, int code_rate, bool has_crc, bool ldro_enabled,
                          bool implicit_header, const uint8_t *d_payloads, const std::vector<size_t> &lengths,
                          uint16_t *d_symbols, size_t symbols_cap) {
    size_t n = 0;
    check(b2s_lora_encode(inst.get(), sf, code_rate, has_crc, ldro_enabled, implicit_header, d_payloads,
                          lengths.data(), lengths.size(), d_symbols, symbols_cap, &n), inst.get());
    return n;
}

// A batch of payloads as the push calls take it: (the bytes back to back, one length per payload)
inline std::pair<std::vector<uint8_t>, std::vector<size_t>> pack_payloads(const std::vector<std::vector<uint8_t>> &payloads) {
    std::pair<std::vector<uint8_t>, std::vector<size_t>> b;
    for (const auto &p : payloads) { b.first.insert(b.first.end(), p.begin(), p.end()); b.second.push_back(p.size()); }
    return b;
}

// ≙ examples/lora/src/transmitter.rs:12-168: a source of Complex<f32> (std::complex<float>) samples; push is the msg
// handler, set_sync_word the synch_word handler (expanded symbols), finish its Pmt::Finished
class LoraTransmitter {
public:
    LoraTransmitter(const Instance &inst, int sf, int code_rate, bool has_crc, bool ldro_enabled, bool implicit_header,
                    size_t oversampling, std::array<uint32_t, 2> sync_symbols, size_t preamble_len, size_t pad)
        : output(inst), inst_(inst) {
        check(b2s_lora_tx_create(inst.get(), sf, code_rate, has_crc, ldro_enabled, implicit_header, oversampling,
                                 sync_symbols.data(), preamble_len, pad, out_ptr(h_)), inst.get());
    }
    void push(const std::vector<std::vector<uint8_t>> &payloads) {
        const auto [bytes, lens] = pack_payloads(payloads);
        check(b2s_lora_tx_push(h_.get(), bytes.data(), lens.data(), lens.size()), inst_.get());
    }
    void set_sync_word(uint32_t s0, uint32_t s1) { check(b2s_lora_tx_set_sync_word(h_.get(), s0, s1), inst_.get()); }
    void finish() { check(b2s_lora_tx_finish(h_.get()), inst_.get()); }
    void reset() { check(b2s_lora_tx_reset(h_.get()), inst_.get()); }
    uint64_t pending() const {
        uint64_t v = 0;
        check(b2s_lora_tx_pending(h_.get(), &v), inst_.get());
        return v;
    }
    // (produced, finished) of one exec into a device slice
    std::pair<size_t, bool> exec(std::complex<float> *d_out, size_t cap) {
        size_t p = 0;
        int32_t f = 0;
        check(b2s_lora_tx_exec(h_.get(), d_out, cap, &p, &f), inst_.get());
        return {p, f != 0};
    }
    void work(WorkIo &io) {
        auto [p, f] = exec(output.slice(), output.capacity());
        output.produce(p);
        if (f) io.finished = true;
    }
    // the burst_start tags since the last drain, in stream order
    std::vector<b2s_lora_burst> drain_bursts() { return drain_records(b2s_lora_tx_drain_bursts, h_.get(), inst_.get()); }
    Writer<std::complex<float>> output;
private:
    const Instance &inst_; Handle<b2s_lora_tx, b2s_lora_tx_destroy> h_;
};

// ≙ examples/wlan/src/{mac,encoder}.rs + the SIGNAL field over a batch from a fresh encoder: frame i is lengths[i]
// bytes of d_payloads (device, back to back) at mcs[i]; 48 subcarrier bytes per OFDM symbol, SIGNAL first, frame after
// frame in d_symbols.  Returns the OFDM symbol total.
inline size_t wlan_encode(const Instance &inst, const std::array<uint8_t, 6> &src, const std::array<uint8_t, 6> &dst,
                          const std::array<uint8_t, 6> &bss, uint32_t sequence_number, uint32_t scrambler_seed,
                          const uint8_t *d_payloads, const std::vector<size_t> &lengths,
                          const std::vector<int32_t> &mcs, uint8_t *d_symbols, size_t symbols_cap) {
    if (mcs.size() != lengths.size()) throw Error(B2S_EINVAL, "wlan_encode: one MCS per payload");
    size_t n = 0;
    check(b2s_wlan_encode(inst.get(), src.data(), dst.data(), bss.data(), sequence_number, scrambler_seed, d_payloads,
                          lengths.data(), mcs.data(), lengths.size(), d_symbols, symbols_cap, &n), inst.get());
    return n;
}

// ≙ examples/wlan/src/bin/tx.rs:44-66 without the radio sink (Mac -> Encoder -> Mapper -> Fft -> Prefix): a source of
// Complex<f32> (std::complex<float>) samples; push is the Mac's tx handler, finish its Pmt::Finished
class WlanTransmitter {
public:
    WlanTransmitter(const Instance &inst, const std::array<uint8_t, 6> &src, const std::array<uint8_t, 6> &dst,
                    const std::array<uint8_t, 6> &bss, int32_t default_mcs, size_t pad_front, size_t pad_tail)
        : output(inst), inst_(inst) {
        check(b2s_wlan_tx_create(inst.get(), src.data(), dst.data(), bss.data(), default_mcs, pad_front, pad_tail,
                                 out_ptr(h_)), inst.get());
    }
    // mcs empty: every frame at the default MCS; otherwise one per payload, -1 meaning the default
    void push(const std::vector<std::vector<uint8_t>> &payloads, const std::vector<int32_t> &mcs = {}) {
        if (!mcs.empty() && mcs.size() != payloads.size()) throw Error(B2S_EINVAL, "wlan push: one MCS per payload");
        const auto [bytes, lens] = pack_payloads(payloads);
        check(b2s_wlan_tx_push(h_.get(), bytes.data(), lens.data(), mcs.empty() ? nullptr : mcs.data(), lens.size()),
              inst_.get());
    }
    void finish() { check(b2s_wlan_tx_finish(h_.get()), inst_.get()); }
    void reset() { check(b2s_wlan_tx_reset(h_.get()), inst_.get()); }
    uint64_t pending() const {
        uint64_t v = 0;
        check(b2s_wlan_tx_pending(h_.get(), &v), inst_.get());
        return v;
    }
    // (produced, finished) of one exec into a device slice
    std::pair<size_t, bool> exec(std::complex<float> *d_out, size_t cap) {
        size_t p = 0;
        int32_t f = 0;
        check(b2s_wlan_tx_exec(h_.get(), d_out, cap, &p, &f), inst_.get());
        return {p, f != 0};
    }
    void work(WorkIo &io) {
        auto [p, f] = exec(output.slice(), output.capacity());
        output.produce(p);
        if (f) io.finished = true;
    }
    // the burst_start tags since the last drain, in stream order
    std::vector<b2s_wlan_burst> drain_bursts() { return drain_records(b2s_wlan_tx_drain_bursts, h_.get(), inst_.get()); }
    Writer<std::complex<float>> output;
private:
    const Instance &inst_; Handle<b2s_wlan_tx, b2s_wlan_tx_destroy> h_;
};

// ≙ examples/zigbee/src/bin/tx.rs:37-56 without the radio sink (Mac -> modulator -> IqDelay): a source of Complex<f32>
// (std::complex<float>) samples; push is the Mac's tx handler and returns how many payloads it dropped for being over
// B2S_ZIGBEE_MAX_PAYLOAD bytes; finish ends the stream after the last frame's tail pad
class ZigbeeTransmitter {
public:
    explicit ZigbeeTransmitter(const Instance &inst, size_t pad = B2S_ZIGBEE_PADDING) : output(inst), inst_(inst) {
        check(b2s_zigbee_tx_create(inst.get(), pad, out_ptr(h_)), inst.get());
    }
    size_t push(const std::vector<std::vector<uint8_t>> &payloads) {
        const auto [bytes, lens] = pack_payloads(payloads);
        size_t dropped = 0;
        check(b2s_zigbee_tx_push(h_.get(), bytes.data(), lens.data(), lens.size(), &dropped), inst_.get());
        return dropped;
    }
    void finish() { check(b2s_zigbee_tx_finish(h_.get()), inst_.get()); }
    void reset() { check(b2s_zigbee_tx_reset(h_.get()), inst_.get()); }
    uint64_t pending() const {
        uint64_t v = 0;
        check(b2s_zigbee_tx_pending(h_.get(), &v), inst_.get());
        return v;
    }
    // (produced, finished) of one exec into a device slice
    std::pair<size_t, bool> exec(std::complex<float> *d_out, size_t cap) {
        size_t p = 0;
        int32_t f = 0;
        check(b2s_zigbee_tx_exec(h_.get(), d_out, cap, &p, &f), inst_.get());
        return {p, f != 0};
    }
    void work(WorkIo &io) {
        auto [p, f] = exec(output.slice(), output.capacity());
        output.produce(p);
        if (f) io.finished = true;
    }
    // the burst_start tags since the last drain, in stream order
    std::vector<b2s_zigbee_burst> drain_bursts() {
        return drain_records(b2s_zigbee_tx_drain_bursts, h_.get(), inst_.get());
    }
    Writer<std::complex<float>> output;
private:
    const Instance &inst_; Handle<b2s_zigbee_tx, b2s_zigbee_tx_destroy> h_;
};

// One input, N outputs moved by one b2s_fanout_exec launch (T: 4- or 8-byte items)
template <typename T, int32_t Deinterleave> class FanOut {
    static_assert(sizeof(T) == 4 || sizeof(T) == 8, "stream fan-out: 4- or 8-byte items");
public:
    FanOut(const Instance &inst, size_t n) : input(inst), inst_(inst), n_(n) {
        if (n == 0) throw Error(B2S_EINVAL, "stream fan-out: at least one output");
        if (n > 256) throw Error(B2S_EUNSUPPORTED, "stream fan-out: at most 256 outputs in one launch");
        for (size_t k = 0; k < n; k++) outs_.push_back(std::make_unique<Writer<T>>(inst));
    }
    Writer<T> &out(size_t k) { return *outs_.at(k); }
    size_t num_outputs() const { return n_; }
    void work(WorkIo &io) {                           // stream_duplicator.rs:66-93, stream_deinterleaver.rs:61-97
        const size_t n_in = input.len();
        size_t cap = SIZE_MAX;
        std::vector<void *> ptrs(n_);
        for (size_t k = 0; k < n_; k++) { cap = std::min(cap, outs_[k]->capacity()); ptrs[k] = outs_[k]->slice(); }
        size_t c = 0, m = 0;
        check(b2s_fanout_exec(inst_.get(), Deinterleave, sizeof(T), input.slice(), n_in, ptrs.data(), n_, cap, &c, &m),
              inst_.get());
        if (m > 0) {
            for (auto &o : outs_) o->produce(m);
            input.consume(c);
        }
        if (Deinterleave ? (n_in - c < n_ && input.finished()) : (n_in - m == 0 && input.finished())) io.finished = true;
    }
    Reader<T> input;
private:
    const Instance &inst_; size_t n_; std::vector<std::unique_ptr<Writer<T>>> outs_;
};
// ≙ blocks::StreamDuplicator<T, N> (stream_duplicator.rs:20-94): outputs[k] = input
template <typename T> using StreamDuplicator = FanOut<T, 0>;
// ≙ blocks::StreamDeinterleaver<T> (stream_deinterleaver.rs:25-98): output[k][j] = input[j N + k], whole groups only
template <typename T> using StreamDeinterleaver = FanOut<T, 1>;

// ---- firdes::hilbert (firdes/basic.rs:202-222), firdes::lowpass (:25-42) and windows::hamming (windows.rs:109-120) ---------------------------
namespace windows {
inline std::vector<double> hamming(size_t len, bool periodic) {
    std::vector<double> w(len);
    if (len) b2s_window_hamming(len, periodic ? 1 : 0, w.data(), len);
    return w;
}
}  // namespace windows
namespace firdes {
inline std::vector<float> hilbert(const std::vector<double> &window) {
    if (window.size() % 2 == 0) throw Error(B2S_EINVAL, "firdes::hilbert: Must be an odd number");   // basic.rs:204
    std::vector<float> t(window.size());
    b2s_firdes_hilbert(window.data(), window.size(), t.data(), t.size());
    return t;
}
inline std::vector<float> lowpass(double cutoff, const std::vector<double> &window) {
    if (!(std::abs(cutoff) < 0.5)) throw Error(B2S_EINVAL, "firdes::lowpass: cutoff must be in ]-1/2, 1/2[");   // :26
    std::vector<float> t(window.size());
    if (!window.empty()) b2s_firdes_lowpass(cutoff, window.data(), window.size(), t.data(), t.size());
    return t;
}
}  // namespace firdes

// ≙ runtime::mocker::Mocker (mocker.rs:33-190): run one block without a scheduler
template <typename Block> class Mocker {
public:
    explicit Mocker(Block &b) : b_(b) {}
    template <typename T> void input(const std::vector<T> &v) { b_.input.set(v); }
    void init_output(size_t n) { b_.output.reserve(n); }
    WorkIo run() {
        WorkIo io;
        for (int guard = 0; guard < (1 << 20); guard++) {
            io = WorkIo{};
            b_.work(io);
            if (io.finished || !io.call_again) break;
        }
        return io;
    }
    auto output() { return b_.output.get(); }
private:
    Block &b_;
};

}  // namespace b2s
