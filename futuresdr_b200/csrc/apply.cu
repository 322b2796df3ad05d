// apply.cu -- element-wise Apply block on the device (src/blocks/apply.rs:100-131).
//
// The reference applies an arbitrary Rust closure `FnMut(&A) -> B` per sample; a device
// backend cannot run host closures, so this is the closed catalogue of the closures that appear
// on the hot path / in the reference's GPU examples (b2s_op).  Stateful closures keep their
// state in device memory: the FM demodulator's `last` sample
// (examples/fm-receiver/src/main.rs:99-104) is the previous input item, so item j reads
// in[j-1] and item 0 reads the carried sample; after the launch the carry is refreshed from
// in[m-1] on the same stream.  The DC blocker's running average is carry.x, read and written by its kernel.  The
// keyfob slicer is the one op with a u8 output, and the SSB transmitter's i16 converter the one that writes two output
// items per input item (ApplyNM<1, 2>, src/blocks/applynm.rs:100-121).
#include <cmath>

#include "chunks.cuh"

struct b2s_apply {
    b2s_ctx *ctx = nullptr;
    b2s_op op = B2S_OP_SCALE_F32;
    float param = 1.0f;
    Buf<float2> d_carry;         // closure state (QUAD_DEMOD*: last sample; DC_BLOCK_F32: .x = the average)
};

namespace {

// arg(v * conj(last)) with num_complex's Mul: re = a.re*b.re - a.im*b.im, im = a.re*b.im + a.im*b.re,
// b = conj(last) = (lr, -li).  __fmul_rn/__fsub_rn keep the products un-fused like the Rust code.
// atan2 in ~30 instructions (CUDA's atan2f is ~60 on its fast path and made the demodulator issue-bound
// at half the HBM roofline): a = min/max of the magnitudes (MUFU.RCP based division), atan(a) = a * P(a^2)
// with a degree-8 minimax P (max error 1.1e-7 rad on [0,1] in f32 Horner form, coefficients fitted in
// scripts -- see DESIGN.md 4.6), then the octant is unfolded with the SIGN BITS so that +-0 behave like
// libm: atan2(+0,-0) = pi, atan2(0,+0) = 0 (the demodulator's first sample multiplies by conj(0)).
// Error <= 4e-7 rad against atan2 in float64 (measured max 3.0e-7 on an H100;
// tests/test_gpu_apply_numerics.py derives the bound).  The special values are libm's: (+-inf, +-inf)
// gives +-pi/4 or +-3pi/4, (+-inf, finite) an axis, and a NaN part NaN.  Three changes keep them (six
// instructions in all), and none changes an output whose parts are finite and at most 2^126:
//   * __fdividef (div.approx.f32) returns 0 for divisors in (2^126, 2^128), so such a pair is scaled
//     by 1/4 first (exact for the divisor; a dividend it pushes into the denormals has a zero quotient);
//   * inf/inf is NaN, so two infinite parts take the quotient 1;
//   * max.NaN / min.NaN keep a NaN part where fmaxf / fminf drop it, and the quotient carries it through.
__device__ __forceinline__ float max_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ float min_nan(float a, float b) {
    float r;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

__device__ __forceinline__ float atan2_poly(float y, float x) {
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx0 = max_nan(ax, ay), mn0 = min_nan(ax, ay);
    const bool big = mx0 > 0x1p126f;
    const float mx = big ? 0.25f * mx0 : mx0, mn = big ? 0.25f * mn0 : mn0;
    const float q = mx <= 0.0f ? 0.0f : __fdividef(mn, mx);
    const float a = mn0 == INFINITY ? 1.0f : q;
    const float s = a * a;
    float p = 0.0029408063273876905f;
    p = fmaf(p, s, -0.0164317823946476f);
    p = fmaf(p, s, 0.04328067600727081f);
    p = fmaf(p, s, -0.07554050534963608f);
    p = fmaf(p, s, 0.10664203763008118f);
    p = fmaf(p, s, -0.14209550619125366f);
    p = fmaf(p, s, 0.19993355870246887f);
    p = fmaf(p, s, -0.33333107829093933f);
    p = fmaf(p, s, 1.0f);
    float r = p * a;
    if (ay > ax) r = 1.57079632679489662f - r;
    if (__float_as_int(x) < 0) r = 3.14159265358979324f - r;
    return copysignf(r, y);
}

__device__ __forceinline__ float quad_demod_one(float2 v, float2 last) {
    const float cr = last.x, ci = -last.y;
    const float pr = __fsub_rn(__fmul_rn(v.x, cr), __fmul_rn(v.y, ci));
    const float pi = __fadd_rn(__fmul_rn(v.x, ci), __fmul_rn(v.y, cr));
    return atan2_poly(pi, pr);
}

template <int OP>
__global__ void apply_kernel(const void *__restrict__ vin, void *__restrict__ vout, long long n, float param,
                             const float2 *__restrict__ carry) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    // four items in flight per thread; nvcc picks 4 by itself except for the demodulators, whose inline asm
    // (max_nan / min_nan) its unroller prices too high
#pragma unroll 4
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        if constexpr (OP == B2S_OP_SCALE_F32) {
            ((float *)vout)[j] = ((const float *)vin)[j] * param;
        } else if constexpr (OP == B2S_OP_SCALE_C32) {
            const float2 v = ((const float2 *)vin)[j];
            ((float2 *)vout)[j] = make_float2(v.x * param, v.y * param);
        } else if constexpr (OP == B2S_OP_QUAD_DEMOD || OP == B2S_OP_QUAD_DEMOD_C32) {
            const float2 *in = (const float2 *)vin;
            const float2 v = in[j];
            const float2 last = (j == 0) ? *carry : in[j - 1];
            const float ph = quad_demod_one(v, last);
            if constexpr (OP == B2S_OP_QUAD_DEMOD) ((float *)vout)[j] = ph;
            else ((float2 *)vout)[j] = make_float2(ph, 0.0f);
        } else if constexpr (OP == B2S_OP_NORM_SQR) {
            const float2 v = ((const float2 *)vin)[j];
            ((float *)vout)[j] = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));   // Complex::norm_sqr
        } else if constexpr (OP == B2S_OP_EXP_F32) {
            ((float *)vout)[j] = expf(((const float *)vin)[j]);
        } else if constexpr (OP == B2S_OP_MAG_C32) {
            const float2 v = ((const float2 *)vin)[j];
            ((float *)vout)[j] = hypotf(v.x, v.y);                                         // Complex::norm
        } else if constexpr (OP == B2S_OP_LOG10_F32) {
            ((float *)vout)[j] = param * log10f(((const float *)vin)[j]);
        } else if constexpr (OP == B2S_OP_DIV_C32) {
            const float2 v = ((const float2 *)vin)[j];
            ((float2 *)vout)[j] = make_float2(__fdiv_rn(v.x, param), __fdiv_rn(v.y, param));   // Complex / f32
        }
    }
}

// B2S_OP_DC_BLOCK_F32: s = (1 - alpha) * s + alpha * x; y = x - s (examples/zigbee/src/bin/rx.rs:70-73).  Only the
// two-operation chain s -> fmul -> fadd is sequential.  One CTA, a three-stage pipeline over chunks of kDcChunk items:
// in phase k the I/O warps stage chunk k (cp.async) and form alpha * x off the chain, lane 0 of warp 0 runs the chain
// over chunk k - 1 (overwriting alpha * x with s), and the I/O warps store x - s of chunk k - 2.
constexpr int kDcChunk = 2048;
__global__ void __launch_bounds__(kThreads)
dc_block_kernel(const float *__restrict__ in, float *__restrict__ out, long long m, float alpha, float oma,
                float2 *__restrict__ carry) {
    __shared__ float xs[3][kDcChunk];
    __shared__ float as[3][kDcChunk];
    const int tid = threadIdx.x;
    const long long nch = (m + kDcChunk - 1) / kDcChunk;
    float s = carry->x;
    for (long long k = 0; k <= nch + 1; k++) {
        if (tid < 32) {
            if (tid == 0 && k >= 1 && k <= nch) {
                float *a = as[(k - 1) % 3];
                const int cnt = (int)min((long long)kDcChunk, m - (k - 1) * kDcChunk);
#pragma unroll 8
                for (int i = 0; i < cnt; i++) {
                    s = __fadd_rn(__fmul_rn(oma, s), a[i]);
                    a[i] = s;
                }
            }
        } else {
            const int t = tid - 32, nt = kThreads - 32;
            if (k < nch) {                                   // stage chunk k
                const long long base = k * kDcChunk;
                const int cnt = (int)min((long long)kDcChunk, m - base);
                float *x = xs[k % 3], *a = as[k % 3];
                for (int i = t; i < cnt; i += nt) cp_async::ca4(x + i, in + base + i);
                cp_async::commit();
                cp_async::wait<0>();
                for (int i = t; i < cnt; i += nt) a[i] = __fmul_rn(alpha, x[i]);   // the thread's own copies
            }
            if (k >= 2) {                                    // store chunk k - 2
                const long long base = (k - 2) * kDcChunk;
                const int cnt = (int)min((long long)kDcChunk, m - base);
                const float *x = xs[(k - 2) % 3], *a = as[(k - 2) % 3];
                for (int i = t; i < cnt; i += nt) out[base + i] = __fsub_rn(x[i], a[i]);
            }
        }
        __syncthreads();
    }
    if (tid == 0) carry->x = s;
}

// B2S_OP_SLICE_F32_U8: x > 0 ? 1 : 0 (examples/keyfob/src/main.rs:73-75).  The chunk split of chunks.cuh with the head
// aligning the OUTPUT to 4 bytes: a chunk's 4 outputs are one 32-bit store, and its 4 inputs one float4 when the input
// (4-byte aligned) is then at 16 bytes, word loads otherwise.
__device__ __forceinline__ unsigned char slice_one(float x) { return x > 0.0f ? 1 : 0; }   // NaN -> 0
__global__ void __launch_bounds__(kThreads)
slice_kernel(const float *__restrict__ in, unsigned char *__restrict__ out, unsigned long long m, unsigned head,
             bool wide) {
    chunk_loop(m, head,
               [&](unsigned long long v) {
                   float r[4];
                   ld_chunk<1>(in + head + 4 * v, wide, r);
                   const unsigned w = (unsigned)slice_one(r[0]) | (unsigned)slice_one(r[1]) << 8 |
                                      (unsigned)slice_one(r[2]) << 16 | (unsigned)slice_one(r[3]) << 24;
                   reinterpret_cast<unsigned *>(out + head)[v] = w;
               },
               [&](unsigned long long i) { out[i] = slice_one(__ldg(in + i)); });
}

// B2S_OP_C32_TO_I16_IQ: (x * param * 32767.0) as i16 per part (examples/ssb/transmit.rs:109-112).  cvt.rzi.s16.f32
// is Rust's `as i16`: it truncates toward zero, clamps to the i16 range and turns NaN into 0.  The pair is one 32-bit
// store when the output is 4-byte aligned, two 16-bit stores otherwise.
__device__ __forceinline__ short to_i16(float x, float param) {
    const float y = __fmul_rn(__fmul_rn(x, param), 32767.0f);
    short r;
    asm("cvt.rzi.s16.f32 %0, %1;" : "=h"(r) : "f"(y));
    return r;
}
__global__ void __launch_bounds__(kThreads)
to_i16_iq_kernel(const float2 *__restrict__ in, short *__restrict__ out, long long n, float param, bool pair32) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        const float2 v = in[j];
        const short re = to_i16(v.x, param), im = to_i16(v.y, param);
        if (pair32) reinterpret_cast<unsigned *>(out)[j] = (unsigned)(unsigned short)re | (unsigned)(unsigned short)im << 16;
        else { out[2 * j] = re; out[2 * j + 1] = im; }
    }
}

template <int OP>
int32_t launch(b2s_apply *a, const void *in, void *out, size_t n) {
    if constexpr (OP == B2S_OP_C32_TO_I16_IQ) {
        b2s_ctx *ctx = a->ctx;
        to_i16_iq_kernel<<<grid_for(ctx, n, 16), kThreads, 0, ctx->stream>>>(
            (const float2 *)in, (short *)out, (long long)n, a->param, ((uintptr_t)out & 3) == 0);
        B2S_CHECK_LAUNCH(ctx);
        return B2S_OK;
    }
    if constexpr (OP == B2S_OP_SLICE_F32_U8) {
        b2s_ctx *ctx = a->ctx;
        const unsigned head = (unsigned)std::min<size_t>(n, (4 - ((uintptr_t)out & 3)) & 3);
        const float *fin = (const float *)in;
        const bool wide = (((uintptr_t)(fin + head)) & 15) == 0;
        slice_kernel<<<grid_for(ctx, std::max<size_t>((n - head) / 4, 1), 16), kThreads, 0, ctx->stream>>>(
            fin, (unsigned char *)out, n, head, wide);
        B2S_CHECK_LAUNCH(ctx);
        return B2S_OK;
    }
    if constexpr (OP == B2S_OP_DC_BLOCK_F32) {
        b2s_ctx *ctx = a->ctx;
        const float oma = 1.0f - a->param;                   // `1.0 - alpha` in f32
        dc_block_kernel<<<1, kThreads, 0, ctx->stream>>>((const float *)in, (float *)out, (long long)n, a->param, oma,
                                                          a->d_carry.get());
        B2S_CHECK_LAUNCH(ctx);
        return B2S_OK;
    }
    b2s_ctx *ctx = a->ctx;
    apply_kernel<OP><<<grid_for(ctx, n, 16), kThreads, 0, ctx->stream>>>(in, out, (long long)n, a->param,
                                                                         a->d_carry.get());
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

bool in_is_complex(b2s_op op) {
    return op == B2S_OP_SCALE_C32 || op == B2S_OP_QUAD_DEMOD || op == B2S_OP_NORM_SQR ||
           op == B2S_OP_QUAD_DEMOD_C32 || op == B2S_OP_MAG_C32 || op == B2S_OP_DIV_C32 || op == B2S_OP_C32_TO_I16_IQ;
}

}  // namespace

extern "C" {

int32_t b2s_apply_create(b2s_ctx *ctx, b2s_op op, float param, b2s_apply **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_apply_create: NULL argument");
    *out = nullptr;
    if ((int)op < 0 || (int)op > (int)B2S_OP_C32_TO_I16_IQ) return b2s_fail(ctx, B2S_EINVAL, "b2s_apply_create: bad op %d", (int)op);
    if (op == B2S_OP_DC_BLOCK_F32 && !std::isfinite(param))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_apply_create: DC blocker alpha %g (a finite value)", (double)param);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_apply> a(new b2s_apply());
    a->ctx = ctx; a->op = op; a->param = param;
    B2S_TRY(a->d_carry.alloc(ctx, 1, "apply state"));
    B2S_TRY(b2s_apply_reset(a.get()));
    *out = a.release();
    return B2S_OK;
}

void b2s_apply_destroy(b2s_apply *a) { PlanDeleter<b2s_apply>()(a); }

// `let mut last = Complex32::new(0.0, 0.0)` (examples/fm-receiver/src/main.rs:98)
int32_t b2s_apply_reset(b2s_apply *a) {
    if (!a) return b2s_fail(nullptr, B2S_EINVAL, "apply is NULL");
    DeviceGuard g(a->ctx->device);
    B2S_CUDA(a->ctx, cudaMemsetAsync(a->d_carry.get(), 0, sizeof(float2), a->ctx->stream));
    return B2S_OK;
}

int32_t b2s_apply_exec(b2s_apply *a, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                       size_t *consumed, size_t *produced) {
    if (!a || !consumed || !produced) return b2s_fail(a ? a->ctx : nullptr, B2S_EINVAL, "b2s_apply_exec: NULL argument");
    const bool iq = a->op == B2S_OP_C32_TO_I16_IQ;                // two i16 items out per c32 item in
    const size_t out_items = iq ? n_out_cap / 2 : n_out_cap;
    const size_t m = n_in < out_items ? n_in : out_items;         // apply.rs:109, applynm.rs:109
    *consumed = m; *produced = iq ? 2 * m : m;
    if (m == 0) return B2S_OK;
    if (!d_in || !d_out) return b2s_fail(a->ctx, B2S_EINVAL, "b2s_apply_exec: NULL buffer");
    // the demodulators read in[j-1] while a neighbour thread writes out[j-1]: the slices must not overlap
    // (the element-wise ops may run in place)
    if (a->op == B2S_OP_DC_BLOCK_F32) {
        if (!word_aligned(d_in) || !word_aligned(d_out))
            return b2s_fail(a->ctx, B2S_EINVAL, "b2s_apply_exec: a slice is not 4-byte aligned");
        if (overlap(d_in, m * sizeof(float), d_out, m * sizeof(float)))
            return b2s_fail(a->ctx, B2S_EINVAL, "b2s_apply_exec: the DC blocker cannot run in place (input and output overlap)");
    }
    if (a->op == B2S_OP_SLICE_F32_U8) {
        if (!word_aligned(d_in)) return b2s_fail(a->ctx, B2S_EINVAL, "b2s_apply_exec: the slicer's input is not 4-byte aligned");
        if (overlap(d_in, m * sizeof(float), d_out, m))
            return b2s_fail(a->ctx, B2S_EINVAL, "b2s_apply_exec: the slicer cannot run in place (input and output overlap)");
    }
    if (iq) {
        if (((uintptr_t)d_in & 7) || ((uintptr_t)d_out & 1))
            return b2s_fail(a->ctx, B2S_EINVAL, "b2s_apply_exec: the i16 converter needs an 8-byte aligned input and a "
                                                "2-byte aligned output");
        if (overlap(d_in, m * sizeof(float2), d_out, m * 2 * sizeof(short)))
            return b2s_fail(a->ctx, B2S_EINVAL, "b2s_apply_exec: the i16 converter cannot run in place (input and output overlap)");
    }
    if (a->op == B2S_OP_QUAD_DEMOD || a->op == B2S_OP_QUAD_DEMOD_C32) {
        if (overlap(d_in, m * sizeof(float2), d_out, m * (a->op == B2S_OP_QUAD_DEMOD ? sizeof(float) : sizeof(float2))))
            return b2s_fail(a->ctx, B2S_EINVAL, "b2s_apply_exec: the quadrature demodulator cannot run in place (input and output overlap)");
    }
    DeviceGuard g(a->ctx->device);
    NvtxRange nvtx("b2s_apply_exec");
    int32_t rc = B2S_EINVAL;
    switch (a->op) {
        case B2S_OP_SCALE_F32: rc = launch<B2S_OP_SCALE_F32>(a, d_in, d_out, m); break;
        case B2S_OP_SCALE_C32: rc = launch<B2S_OP_SCALE_C32>(a, d_in, d_out, m); break;
        case B2S_OP_QUAD_DEMOD: rc = launch<B2S_OP_QUAD_DEMOD>(a, d_in, d_out, m); break;
        case B2S_OP_NORM_SQR: rc = launch<B2S_OP_NORM_SQR>(a, d_in, d_out, m); break;
        case B2S_OP_QUAD_DEMOD_C32: rc = launch<B2S_OP_QUAD_DEMOD_C32>(a, d_in, d_out, m); break;
        case B2S_OP_EXP_F32: rc = launch<B2S_OP_EXP_F32>(a, d_in, d_out, m); break;
        case B2S_OP_MAG_C32: rc = launch<B2S_OP_MAG_C32>(a, d_in, d_out, m); break;
        case B2S_OP_LOG10_F32: rc = launch<B2S_OP_LOG10_F32>(a, d_in, d_out, m); break;
        case B2S_OP_DC_BLOCK_F32: rc = launch<B2S_OP_DC_BLOCK_F32>(a, d_in, d_out, m); break;
        case B2S_OP_SLICE_F32_U8: rc = launch<B2S_OP_SLICE_F32_U8>(a, d_in, d_out, m); break;
        case B2S_OP_DIV_C32: rc = launch<B2S_OP_DIV_C32>(a, d_in, d_out, m); break;
        case B2S_OP_C32_TO_I16_IQ: rc = launch<B2S_OP_C32_TO_I16_IQ>(a, d_in, d_out, m); break;
    }
    if (rc != B2S_OK) return rc;
    if (a->op == B2S_OP_QUAD_DEMOD || a->op == B2S_OP_QUAD_DEMOD_C32) {
        // last = in[m-1] for the next call (stream-ordered after the kernel that read the old carry)
        B2S_CUDA(a->ctx, cudaMemcpyAsync(a->d_carry.get(), (const float2 *)d_in + (m - 1), sizeof(float2),
                                         cudaMemcpyDeviceToDevice, a->ctx->stream));
    }
    (void)in_is_complex;
    return B2S_OK;
}

}  // extern "C"
