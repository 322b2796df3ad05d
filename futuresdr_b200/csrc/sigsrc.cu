// sigsrc.cu -- blocks::SignalSource (src/blocks/signal_source/mod.rs:29-227) with its fixed-point NCO
// (fxpt_nco.rs:3-43) and FixedPointPhase (fxpt_phase.rs:8-99).
//
// The NCO's phase is a wrapping 32-bit integer, so the phase of output k of a call is exactly phase0 + k * inc
// (mod 2^32): every output is independent, and one data-parallel kernel writes bit-identical samples at any stream
// length.  The plan keeps phase and inc on the host (they depend only on counts), so calls are stream-ordered and
// never synchronise.
//
// The sine table (1024 x {slope, offset}) is regenerated from its formula, evaluated in f64 and rounded to f32:
//     f(u) = sin(u pi / 2^31),  incx = (2^32 - 1) / 1024,  a = i incx,  b = (i + 1) incx
//     T[i] = ((f(b) - f(a)) / (b - a), f(a))
// which reproduces every one of the reference's 2048 literals (fxpt_phase.rs:101-1126).
#include <cmath>
#include <cstdint>

#include "chunks.cuh"

namespace {

constexpr int kTableN = 1024;
constexpr int kTablePad = kTableN + kTableN / 32;    // one pad word per 32 entries, see tpos()
constexpr uint32_t kAccumMask = 0x3FFFFFu;           // ACCUM_MASK: 32 - 10 fraction bits (fxpt_phase.rs:70)

struct SineTable { float slope[kTableN], offset[kTableN]; };

const SineTable &sine_table() {
    static const SineTable t = [] {
        SineTable s;
        const double incx = (4294967296.0 - 1.0) / kTableN;
        auto f = [](double u) { return std::sin(u * M_PI / 2147483648.0); };
        for (int i = 0; i < kTableN; i++) {
            const double a = i * incx, b = (i + 1) * incx;
            s.slope[i] = (float)((f(b) - f(a)) / (b - a));
            s.offset[i] = (float)f(a);
        }
        return s;
    }();
    return t;
}

// Rust's `as i32` from f32: truncation toward zero, saturating, NaN -> 0
int32_t rust_as_i32(float v) {
    if (v != v) return 0;
    if (v >= 2147483648.0f) return INT32_MAX;
    if (v <= -2147483648.0f) return INT32_MIN;
    return (int32_t)v;
}

constexpr float kPi = 3.14159265358979323846f;       // std::f32::consts::PI
constexpr float kTau = 6.28318530717958647692f;      // std::f32::consts::TAU

// FixedPointPhase::new (fxpt_phase.rs:75-82): f32 operations in the reference's order (the library is built with
// -ffp-contract=off, so nothing here is fused)
int32_t fxpt_phase_new(float x) {
    const float q = x / kTau + 0.5f;
    const int32_t d = rust_as_i32(std::floor(q));
    const float xr = x - (float)d * kTau;
    return rust_as_i32(xr * 2147483648.0f / kPi);
}

float fxpt_eval(uint32_t ux) {                       // fxpt_phase.rs:85-98 after the index is formed
    const SineTable &t = sine_table();
    const uint32_t i = ux >> 22;
    const float m = t.slope[i] * (float)(ux & kAccumMask);
    return m + t.offset[i];
}

// The sample before the amplitude is always finite, so a NaN output comes from the amplitude alone.  The GPU
// returns one canonical NaN (0x7FFFFFFF); the reference's f32 multiply on x86-64 (SSE mulss) returns a NaN operand
// quieted, and the default NaN 0xFFC00000 for 0 * inf.  The kernel writes these bits in place of any NaN result.
uint32_t x86_nan_of_product(float amp) {
    uint32_t b;
    std::memcpy(&b, &amp, sizeof b);
    return amp != amp ? b | 0x00400000u : 0xFFC00000u;
}

// Entry i of each half of the table lives at i + i / 32 in shared memory.  Lanes of a warp read entries a fixed
// stride apart; without the pad a stride that is a multiple of 32 entries (frequency = fs/64 gives 64 entries per
// f32 thread) puts every lane on one bank.  With it, stride 32 m spreads over 32 / gcd(m, 32) banks.
__device__ __forceinline__ unsigned tpos(unsigned i) { return i + (i >> 5); }

// Float j of the call's output: sample j (f32) or component j & 1 of sample j >> 1 (Complex32).
template <int WAVE, bool CPLX>
__device__ __forceinline__ float sample_float(unsigned long long j, uint32_t phase0, uint32_t inc, float amp,
                                              uint32_t nan_bits, const float *sl, const float *of) {
    const unsigned long long k = CPLX ? j >> 1 : j;
    const uint32_t ph = phase0 + (uint32_t)k * inc;                     // NCO::step, wrapping (fxpt_phase.rs:51-55)
    const bool im = CPLX && (j & 1);
    float v;
    if constexpr (WAVE == B2S_WAVE_SQUARE) {
        if constexpr (!CPLX) v = (int32_t)ph < 0 ? 1.0f : 0.0f;         // mod.rs:161-163
        else {                                                          // value >> 30: -2 (1,0) -1 (1,1) 0 (0,1) 1 (0,0)
            const uint32_t b31 = ph >> 31, b30 = (ph >> 30) & 1u;
            v = (im ? b31 == b30 : b31 != 0) ? 1.0f : 0.0f;             // mod.rs:213-221
        }
    } else {
        const bool use_cos = CPLX ? !im : WAVE == B2S_WAVE_COS;         // Complex32: (cos, sin) for sin and cos alike
        const uint32_t ux = use_cos ? ph + 0x40000000u : ph;
        const unsigned i = tpos(ux >> 22);
        v = __fadd_rn(__fmul_rn(sl[i], __uint2float_rn(ux & kAccumMask)), of[i]);
    }
    const float r = __fmul_rn(v, amp);                                  // `a * self.amplitude` (mod.rs:99)
    return r != r ? __uint_as_float(nan_bits) : r;
}

// Writes nf floats at out on the aligned-chunk loop (chunks.cuh), counted in floats; `head` brings out to 16 bytes,
// so every chunk is one float4 store.
template <int WAVE, bool CPLX>
__global__ void __launch_bounds__(kThreads)
sigsrc_kernel(float *__restrict__ out, unsigned long long nf, unsigned head, uint32_t phase0, uint32_t inc, float amp,
              uint32_t nan_bits, const float *__restrict__ table) {
    __shared__ float sl[kTablePad], of[kTablePad];
    if constexpr (WAVE != B2S_WAVE_SQUARE) {
        for (int i = threadIdx.x; i < kTableN; i += kThreads) {
            sl[tpos(i)] = __ldg(table + i);
            of[tpos(i)] = __ldg(table + kTableN + i);
        }
        __syncthreads();
    }
    float4 *ov = reinterpret_cast<float4 *>(out + head);
    chunk_loop(nf, head, [&](unsigned long long v) {
        const unsigned long long j = head + 4 * v;
        float4 r;
        r.x = sample_float<WAVE, CPLX>(j, phase0, inc, amp, nan_bits, sl, of);
        r.y = sample_float<WAVE, CPLX>(j + 1, phase0, inc, amp, nan_bits, sl, of);
        r.z = sample_float<WAVE, CPLX>(j + 2, phase0, inc, amp, nan_bits, sl, of);
        r.w = sample_float<WAVE, CPLX>(j + 3, phase0, inc, amp, nan_bits, sl, of);
        ov[v] = r;
    }, [&](unsigned long long j) { out[j] = sample_float<WAVE, CPLX>(j, phase0, inc, amp, nan_bits, sl, of); });
}

template <int WAVE, bool CPLX>
void launch(unsigned grid, cudaStream_t st, float *out, unsigned long long nf, unsigned head, uint32_t phase0,
            uint32_t inc, float amp, uint32_t nan_bits, const float *table) {
    sigsrc_kernel<WAVE, CPLX><<<grid, kThreads, 0, st>>>(out, nf, head, phase0, inc, amp, nan_bits, table);
}

}  // namespace

struct b2s_sigsrc {
    b2s_ctx *ctx = nullptr;
    b2s_wave wave = B2S_WAVE_SIN;
    bool cplx = false;
    uint32_t phase = 0, inc = 0;       // NCO (fxpt_nco.rs:5-9), advanced by each exec
    float amplitude = 0.0f;
    Buf<SineTable> d_table;            // slope[1024] then offset[1024]
};

extern "C" {

int32_t b2s_fxpt_phase_new(float x, int32_t *value) {
    if (!value) return b2s_fail(nullptr, B2S_EINVAL, "b2s_fxpt_phase_new: value is NULL");
    *value = fxpt_phase_new(x);
    return B2S_OK;
}

int32_t b2s_fxpt_sin_cos(int32_t value, float *sin_out, float *cos_out) {
    if (!sin_out || !cos_out) return b2s_fail(nullptr, B2S_EINVAL, "b2s_fxpt_sin_cos: NULL argument");
    *sin_out = fxpt_eval((uint32_t)value);
    *cos_out = fxpt_eval((uint32_t)value + 0x40000000u);
    return B2S_OK;
}

int32_t b2s_sigsrc_create(b2s_ctx *ctx, b2s_wave wave, int32_t complex_items, float frequency, float sample_rate,
                          float amplitude, float initial_phase, b2s_sigsrc **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_sigsrc_create: NULL argument");
    *out = nullptr;
    if (wave != B2S_WAVE_COS && wave != B2S_WAVE_SIN && wave != B2S_WAVE_SQUARE)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_sigsrc_create: wave %d is not COS, SIN or SQUARE", (int)wave);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_sigsrc> s(new b2s_sigsrc());
    s->ctx = ctx;
    s->wave = wave;
    s->cplx = complex_items != 0;
    s->amplitude = amplitude;
    // NCO::new(initial_phase, 2.0 * PI * frequency / sample_rate) (mod.rs:130-133); no argument is validated
    const float two_pi = 2.0f * kPi;
    const float w = two_pi * frequency;
    s->phase = (uint32_t)fxpt_phase_new(initial_phase);
    s->inc = (uint32_t)fxpt_phase_new(w / sample_rate);
    B2S_TRY(s->d_table.upload(ctx, &sine_table(), 1, "sigsrc table"));
    *out = s.release();
    return B2S_OK;
}

void b2s_sigsrc_destroy(b2s_sigsrc *s) { PlanDeleter<b2s_sigsrc>()(s); }

int32_t b2s_sigsrc_set_amplitude(b2s_sigsrc *s, float amplitude) {
    if (!s) return b2s_fail(nullptr, B2S_EINVAL, "sigsrc is NULL");
    s->amplitude = amplitude;
    return B2S_OK;
}

int32_t b2s_sigsrc_phase(const b2s_sigsrc *s, int32_t *value, int32_t *inc) {
    if (!s || !value || !inc) return b2s_fail(s ? s->ctx : nullptr, B2S_EINVAL, "b2s_sigsrc_phase: NULL argument");
    *value = (int32_t)s->phase;
    *inc = (int32_t)s->inc;
    return B2S_OK;
}

int32_t b2s_sigsrc_exec(b2s_sigsrc *s, void *d_out, size_t n_out_cap, size_t *produced) {
    if (!s || !produced) return b2s_fail(s ? s->ctx : nullptr, B2S_EINVAL, "b2s_sigsrc_exec: NULL argument");
    *produced = 0;
    if (n_out_cap == 0) return B2S_OK;
    if (!d_out) return b2s_fail(s->ctx, B2S_EINVAL, "b2s_sigsrc_exec: NULL output");
    if (!word_aligned(d_out)) return b2s_fail(s->ctx, B2S_EINVAL, "b2s_sigsrc_exec: output is not 4-byte aligned");
    DeviceGuard g(s->ctx->device);
    NvtxRange nvtx("b2s_sigsrc_exec");
    const unsigned long long nf = (unsigned long long)n_out_cap * (s->cplx ? 2 : 1);
    const unsigned head = (unsigned)std::min<unsigned long long>(head_items(d_out, 4), nf);
    const unsigned grid = grid_for(s->ctx, (nf - head) / 4);
    float *o = (float *)d_out;
    cudaStream_t st = s->ctx->stream;
    const uint32_t ph = s->phase, inc = s->inc;
    const float amp = s->amplitude;
    const uint32_t nan_bits = x86_nan_of_product(amp);
    const float *table = reinterpret_cast<const float *>(s->d_table.get());
    switch (s->wave * 2 + (s->cplx ? 1 : 0)) {
        case B2S_WAVE_COS * 2: launch<B2S_WAVE_COS, false>(grid, st, o, nf, head, ph, inc, amp, nan_bits, table); break;
        case B2S_WAVE_SIN * 2: launch<B2S_WAVE_SIN, false>(grid, st, o, nf, head, ph, inc, amp, nan_bits, table); break;
        case B2S_WAVE_SQUARE * 2: launch<B2S_WAVE_SQUARE, false>(grid, st, o, nf, head, ph, inc, amp, nan_bits, table); break;
        case B2S_WAVE_COS * 2 + 1:                      // Complex32 cos is sin (mod.rs:175-182)
        case B2S_WAVE_SIN * 2 + 1: launch<B2S_WAVE_SIN, true>(grid, st, o, nf, head, ph, inc, amp, nan_bits, table); break;
        default: launch<B2S_WAVE_SQUARE, true>(grid, st, o, nf, head, ph, inc, amp, nan_bits, table); break;
    }
    B2S_CHECK_LAUNCH(s->ctx);
    s->phase += (uint32_t)n_out_cap * s->inc;           // n steps of the NCO, wrapping
    *produced = n_out_cap;
    return B2S_OK;
}

}  // extern "C"
