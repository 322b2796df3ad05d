// stream.cu -- the stream-plumbing blocks of branching flowgraphs: Combine (src/blocks/combine.rs:102-136), Split
// (split.rs:95-126), StreamDuplicator (stream_duplicator.rs:66-93) and StreamDeinterleaver
// (stream_deinterleaver.rs:61-97).  Delay (delay.rs) needs no kernel: pad is b2s_memset, copy b2s_memcpy_d2d.
//
// Every kernel is element-wise or a permutation, so each is bound by HBM traffic.  Items are handled as 32-bit
// words (f32 = 1 word, Complex32 / f64 = 2 words), so any 4-byte-aligned slice works.  Element-wise kernels run on
// the aligned-chunk loop of chunks.cuh; Combine and Split take the head from output 0, the duplicator from its input.
//
// Bit-exactness: every closure is written with __fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn in the order of the
// Rust expression (Rust does not contract to FMA; the library is also built with -ffp-contract=off).  norm() is
// glibc's hypotf, which for finite inputs equals (float)sqrt((double)x*x + (double)y*y): the squares are exact in
// f64, the sum and the square root are rounded once each, then one rounding to f32.  hypotf(+-inf, anything) = +inf,
// NaN included, so an infinite component is tested first.
#include <algorithm>
#include <cstdint>

#include "chunks.cuh"

namespace {

constexpr int kMaxOuts = 256;                // output pointers passed in the kernel parameter block (2 KiB)
constexpr size_t kTileBytes = 16384;         // deinterleave: target shared-memory tile

// ---- Combine closures: words per item of in0, in1, out and the closure itself ---------------------------------
template <int OP> struct CombineOp;
template <> struct CombineOp<B2S_COMBINE_ADD_F32> {         // a + b (tests/combine.rs)
    static constexpr int WA = 1, WB = 1, WO = 1;
    __device__ static void f(const float *a, const float *b, float *o) { o[0] = __fadd_rn(a[0], b[0]); }
};
template <> struct CombineOp<B2S_COMBINE_SUB_F32> {         // i1 - i2 (m17)
    static constexpr int WA = 1, WB = 1, WO = 1;
    __device__ static void f(const float *a, const float *b, float *o) { o[0] = __fsub_rn(a[0], b[0]); }
};
template <> struct CombineOp<B2S_COMBINE_MUL_F32> {         // a * b (cw)
    static constexpr int WA = 1, WB = 1, WO = 1;
    __device__ static void f(const float *a, const float *b, float *o) { o[0] = __fmul_rn(a[0], b[0]); }
};
template <> struct CombineOp<B2S_COMBINE_CONJ_MUL_C32> {    // a * b.conj(), num_complex Mul with other = (b.re, -b.im)
    static constexpr int WA = 2, WB = 2, WO = 2;
    __device__ static void f(const float *a, const float *b, float *o) {
        const float cr = b[0], ci = -b[1];
        const float re = __fsub_rn(__fmul_rn(a[0], cr), __fmul_rn(a[1], ci));
        const float im = __fadd_rn(__fmul_rn(a[0], ci), __fmul_rn(a[1], cr));
        o[0] = re; o[1] = im;
    }
};
template <> struct CombineOp<B2S_COMBINE_MAG_DIV_C32_F32> { // a.norm() / b (wlan)
    static constexpr int WA = 2, WB = 1, WO = 1;
    __device__ static void f(const float *a, const float *b, float *o) {
        const float x = a[0], y = a[1];
        float n;
        if (isinf(x) || isinf(y)) n = __int_as_float(0x7F800000);
        else n = __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn((double)x, (double)x), __dmul_rn((double)y, (double)y))));
        o[0] = __fdiv_rn(n, b[0]);
    }
};
template <> struct CombineOp<B2S_COMBINE_TO_C32> {          // Complex32::new(i, q) (ssb USB)
    static constexpr int WA = 1, WB = 1, WO = 2;
    __device__ static void f(const float *a, const float *b, float *o) { o[0] = a[0]; o[1] = b[0]; }
};
template <> struct CombineOp<B2S_COMBINE_TO_C32_NEG_Q> {    // Complex32::new(i, q * -1.0) (ssb LSB): a multiply
    static constexpr int WA = 1, WB = 1, WO = 2;
    __device__ static void f(const float *a, const float *b, float *o) { o[0] = a[0]; o[1] = __fmul_rn(b[0], -1.0f); }
};

template <int OP>
__global__ void __launch_bounds__(kThreads)
combine_kernel(const float *__restrict__ a, const float *__restrict__ b, float *__restrict__ o, unsigned long long m,
               unsigned head) {
    using Op = CombineOp<OP>;
    constexpr int WA = Op::WA, WB = Op::WB, WO = Op::WO;
    const float *a0 = a + (size_t)head * WA, *b0 = b + (size_t)head * WB;
    float *o0 = o + (size_t)head * WO;
    const bool wa = aligned16(a0), wb = aligned16(b0), wo = aligned16(o0);
    chunk_loop(m, head, [&](unsigned long long v) {
        float ra[4 * WA], rb[4 * WB], ro[4 * WO];
        ld_chunk<WA>(a0 + 4 * WA * v, wa, ra);
        ld_chunk<WB>(b0 + 4 * WB * v, wb, rb);
#pragma unroll
        for (int k = 0; k < 4; k++) Op::f(ra + k * WA, rb + k * WB, ro + k * WO);
        st_chunk<WO>(o0 + 4 * WO * v, wo, ro);
    }, [&](unsigned long long i) {
        float ra[WA], rb[WB], ro[WO];
        for (int j = 0; j < WA; j++) ra[j] = a[i * WA + j];
        for (int j = 0; j < WB; j++) rb[j] = b[i * WB + j];
        Op::f(ra, rb, ro);
        for (int j = 0; j < WO; j++) o[i * WO + j] = ro[j];
    });
}

// ---- Split closures -------------------------------------------------------------------------------------------
template <int OP> struct SplitOp;
template <> struct SplitOp<B2S_SPLIT_RE_IM> {               // |a| (a.re, a.im) (tests/split.rs)
    static constexpr int WI = 2;
    __device__ static void f(const float *x, float &y0, float &y1) { y0 = x[0]; y1 = x[1]; }
};
template <> struct SplitOp<B2S_SPLIT_DUP_F32> {             // |v| (v, v) (ssb)
    static constexpr int WI = 1;
    __device__ static void f(const float *x, float &y0, float &y1) { y0 = x[0]; y1 = x[0]; }
};

template <int OP>
__global__ void __launch_bounds__(kThreads)
split_kernel(const float *__restrict__ in, float *__restrict__ o0, float *__restrict__ o1, unsigned long long m,
             unsigned head) {
    using Op = SplitOp<OP>;
    constexpr int WI = Op::WI;
    const float *i0 = in + (size_t)head * WI;
    float *p0 = o0 + head, *p1 = o1 + head;
    const bool wi = aligned16(i0), w0 = aligned16(p0), w1 = aligned16(p1);
    chunk_loop(m, head, [&](unsigned long long v) {
        float r[4 * WI], y0[4], y1[4];
        ld_chunk<WI>(i0 + 4 * WI * v, wi, r);
#pragma unroll
        for (int k = 0; k < 4; k++) Op::f(r + k * WI, y0[k], y1[k]);
        st_chunk<1>(p0 + 4 * v, w0, y0);
        st_chunk<1>(p1 + 4 * v, w1, y1);
    }, [&](unsigned long long i) {
        float y0, y1;
        Op::f(in + i * WI, y0, y1);
        o0[i] = y0;
        o1[i] = y1;
    });
}

// ---- fan-out: N output pointers in the parameter block --------------------------------------------------------
struct OutPtrs { float *p[kMaxOuts]; };

// StreamDuplicator: a copy, so items of any width are moved as 32-bit words.  Every thread loads one 4-word chunk of
// the input once and stores it to all N outputs.
__global__ void __launch_bounds__(kThreads)
duplicate_kernel(const float *__restrict__ in, const OutPtrs outs, int n_outs, unsigned long long m, unsigned head) {
    const float *i0 = in + head;
    const bool wi = aligned16(i0);
    chunk_loop(m, head, [&](unsigned long long v) {
        float r[4];
        ld_chunk<1>(i0 + 4 * v, wi, r);
        for (int k = 0; k < n_outs; k++) {
            float *ok = outs.p[k] + head;
            st_chunk<1>(ok + 4 * v, aligned16(ok), r);
        }
    }, [&](unsigned long long i) {
        const float r = in[i];
        for (int k = 0; k < n_outs; k++) outs.p[k][i] = r;
    });
}

// StreamDeinterleaver: one CTA per tile of G groups of N items.  The tile is read contiguously (float4 when the input
// is 16-byte aligned) into shared memory, one row of N*W words per group at an odd row stride S, so that the column
// reads of the write phase (group j = consecutive lanes) fall on distinct banks.  Output k then receives its G items
// as one contiguous run of stores.
__global__ void __launch_bounds__(kThreads)
deinterleave_kernel(const float *__restrict__ in, const OutPtrs outs, int n, int w, unsigned long long m, int G,
                    int S) {
    extern __shared__ float tile[];
    const unsigned long long g0 = (unsigned long long)blockIdx.x * G;
    const int gc = (int)min((unsigned long long)G, m - g0);              // groups in this tile
    const int row = n * w;                                               // words per group
    const int nwords = gc * row;
    const float *src = in + g0 * row;
    if (aligned16(src) && (row & 3) == 0) {                              // whole float4s per group, aligned start
        for (int q = threadIdx.x; q < nwords / 4; q += kThreads) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(src) + q);
            const int p = 4 * q, j = p / row, r = p - j * row;           // 4 | row: the float4 stays in one row
            float *d = tile + j * S + r;
            d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
        }
    } else {
        for (int p = threadIdx.x; p < nwords; p += kThreads) {
            const int j = p / row;
            tile[j * S + (p - j * row)] = __ldg(src + p);
        }
    }
    __syncthreads();
    const int per_out = gc * w;                                          // words each output receives from this tile
    for (int e = threadIdx.x; e < n * per_out; e += kThreads) {
        const int k = e / per_out, rem = e - k * per_out, j = rem / w, c = rem - j * w;
        outs.p[k][g0 * w + rem] = tile[j * S + k * w + c];
    }
}

// ---- host side ------------------------------------------------------------------------------------------------
struct CombineTypes { size_t a, b, o; };
CombineTypes combine_types(b2s_combine_op op) {
    switch (op) {
        case B2S_COMBINE_CONJ_MUL_C32: return {8, 8, 8};
        case B2S_COMBINE_MAG_DIV_C32_F32: return {8, 4, 4};
        case B2S_COMBINE_TO_C32:
        case B2S_COMBINE_TO_C32_NEG_Q: return {4, 4, 8};
        default: return {4, 4, 4};
    }
}

template <int OP> void launch_combine(b2s_ctx *ctx, const void *a, const void *b, void *o, size_t m) {
    const unsigned head = (unsigned)std::min<size_t>(head_items(o, combine_types((b2s_combine_op)OP).o), m);
    combine_kernel<OP><<<grid_for(ctx, (m - head) / 4), kThreads, 0, ctx->stream>>>(
        (const float *)a, (const float *)b, (float *)o, m, head);
}

template <int OP> void launch_split(b2s_ctx *ctx, const void *in, void *o0, void *o1, size_t m) {
    const unsigned head = (unsigned)std::min<size_t>(head_items(o0, 4), m);
    split_kernel<OP><<<grid_for(ctx, (m - head) / 4), kThreads, 0, ctx->stream>>>(
        (const float *)in, (float *)o0, (float *)o1, m, head);
}

}  // namespace

extern "C" {

int32_t b2s_combine_exec(b2s_ctx *ctx, b2s_combine_op op, const void *d_in0, size_t n_in0, const void *d_in1,
                         size_t n_in1, void *d_out, size_t n_out_cap, size_t *consumed, size_t *produced) {
    if (!ctx || !consumed || !produced) return b2s_fail(ctx, B2S_EINVAL, "b2s_combine_exec: NULL argument");
    *consumed = *produced = 0;
    if ((unsigned)op > (unsigned)B2S_COMBINE_TO_C32_NEG_Q)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_combine_exec: op %d is not a b2s_combine_op", (int)op);
    const size_t m = std::min(std::min(n_in0, n_in1), n_out_cap);        // combine.rs:114-115
    if (m == 0) return B2S_OK;
    if (!d_in0 || !d_in1 || !d_out) return b2s_fail(ctx, B2S_EINVAL, "b2s_combine_exec: NULL slice");
    if (!word_aligned(d_in0) || !word_aligned(d_in1) || !word_aligned(d_out))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_combine_exec: a slice is not 4-byte aligned");
    const CombineTypes t = combine_types(op);
    if (bad_alias(d_out, m * t.o, t.o, d_in0, m * t.a, t.a) || bad_alias(d_out, m * t.o, t.o, d_in1, m * t.b, t.b))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_combine_exec: the output overlaps an input other than exactly in place");
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_combine_exec");
    switch (op) {
        case B2S_COMBINE_ADD_F32: launch_combine<B2S_COMBINE_ADD_F32>(ctx, d_in0, d_in1, d_out, m); break;
        case B2S_COMBINE_SUB_F32: launch_combine<B2S_COMBINE_SUB_F32>(ctx, d_in0, d_in1, d_out, m); break;
        case B2S_COMBINE_MUL_F32: launch_combine<B2S_COMBINE_MUL_F32>(ctx, d_in0, d_in1, d_out, m); break;
        case B2S_COMBINE_CONJ_MUL_C32: launch_combine<B2S_COMBINE_CONJ_MUL_C32>(ctx, d_in0, d_in1, d_out, m); break;
        case B2S_COMBINE_MAG_DIV_C32_F32: launch_combine<B2S_COMBINE_MAG_DIV_C32_F32>(ctx, d_in0, d_in1, d_out, m); break;
        case B2S_COMBINE_TO_C32: launch_combine<B2S_COMBINE_TO_C32>(ctx, d_in0, d_in1, d_out, m); break;
        default: launch_combine<B2S_COMBINE_TO_C32_NEG_Q>(ctx, d_in0, d_in1, d_out, m); break;
    }
    B2S_CHECK_LAUNCH(ctx);
    *consumed = *produced = m;
    return B2S_OK;
}

int32_t b2s_split_exec(b2s_ctx *ctx, b2s_split_op op, const void *d_in, size_t n_in, void *d_out0, void *d_out1,
                       size_t n_out_cap, size_t *consumed, size_t *produced) {
    if (!ctx || !consumed || !produced) return b2s_fail(ctx, B2S_EINVAL, "b2s_split_exec: NULL argument");
    *consumed = *produced = 0;
    if (op != B2S_SPLIT_RE_IM && op != B2S_SPLIT_DUP_F32)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_split_exec: op %d is not a b2s_split_op", (int)op);
    const size_t m = std::min(n_in, n_out_cap);                          // split.rs:106-107
    if (m == 0) return B2S_OK;
    if (!d_in || !d_out0 || !d_out1) return b2s_fail(ctx, B2S_EINVAL, "b2s_split_exec: NULL slice");
    if (!word_aligned(d_in) || !word_aligned(d_out0) || !word_aligned(d_out1))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_split_exec: a slice is not 4-byte aligned");
    const size_t ib = op == B2S_SPLIT_RE_IM ? 8 : 4;
    if (bad_alias(d_out0, 4 * m, 4, d_in, ib * m, ib) || bad_alias(d_out1, 4 * m, 4, d_in, ib * m, ib) ||
        overlap(d_out0, 4 * m, d_out1, 4 * m))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_split_exec: outputs overlap each other or the input other than in place");
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_split_exec");
    if (op == B2S_SPLIT_RE_IM) launch_split<B2S_SPLIT_RE_IM>(ctx, d_in, d_out0, d_out1, m);
    else launch_split<B2S_SPLIT_DUP_F32>(ctx, d_in, d_out0, d_out1, m);
    B2S_CHECK_LAUNCH(ctx);
    *consumed = *produced = m;
    return B2S_OK;
}

int32_t b2s_fanout_exec(b2s_ctx *ctx, int32_t deinterleave, size_t item_bytes, const void *d_in, size_t n_in,
                        void *const *d_outs, size_t n_outs, size_t n_out_cap, size_t *consumed, size_t *produced) {
    if (!ctx || !consumed || !produced) return b2s_fail(ctx, B2S_EINVAL, "b2s_fanout_exec: NULL argument");
    *consumed = *produced = 0;
    if (item_bytes != 4 && item_bytes != 8)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_fanout_exec: items of %zu bytes (4 or 8 supported)", item_bytes);
    if (n_outs == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_fanout_exec: no outputs");
    if (n_outs > (size_t)kMaxOuts)
        return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_fanout_exec: %zu outputs (at most %d)", n_outs, kMaxOuts);
    const size_t m = deinterleave ? std::min(n_out_cap, n_in / n_outs)   // stream_deinterleaver.rs:75
                                  : std::min(n_out_cap, n_in);           // stream_duplicator.rs:80
    if (m == 0) return B2S_OK;
    if (!d_in || !d_outs) return b2s_fail(ctx, B2S_EINVAL, "b2s_fanout_exec: NULL slice");
    const size_t in_items = deinterleave ? m * n_outs : m;
    if (!word_aligned(d_in)) return b2s_fail(ctx, B2S_EINVAL, "b2s_fanout_exec: input is not 4-byte aligned");
    OutPtrs ptrs{};
    std::vector<std::pair<uintptr_t, size_t>> spans;
    for (size_t k = 0; k < n_outs; k++) {
        if (!d_outs[k]) return b2s_fail(ctx, B2S_EINVAL, "b2s_fanout_exec: output %zu is NULL", k);
        if (!word_aligned(d_outs[k])) return b2s_fail(ctx, B2S_EINVAL, "b2s_fanout_exec: output %zu is not 4-byte aligned", k);
        if (overlap(d_outs[k], m * item_bytes, d_in, in_items * item_bytes))
            return b2s_fail(ctx, B2S_EINVAL, "b2s_fanout_exec: output %zu overlaps the input", k);
        ptrs.p[k] = (float *)d_outs[k];
        spans.push_back({(uintptr_t)d_outs[k], k});
    }
    std::sort(spans.begin(), spans.end());
    for (size_t k = 1; k < spans.size(); k++)
        if (spans[k].first < spans[k - 1].first + m * item_bytes)
            return b2s_fail(ctx, B2S_EINVAL, "b2s_fanout_exec: outputs %zu and %zu overlap", spans[k - 1].second, spans[k].second);
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_fanout_exec");
    const int w = (int)(item_bytes / 4);
    if (!deinterleave) {
        const size_t words = m * w;
        const unsigned head = (unsigned)std::min<size_t>(head_items(d_in, 4), words);
        duplicate_kernel<<<grid_for(ctx, (words - head) / 4), kThreads, 0, ctx->stream>>>((const float *)d_in, ptrs,
                                                                                         (int)n_outs, words, head);
    } else {
        const size_t row = n_outs * w;                                   // words per group
        const size_t G = std::max<size_t>(32, kTileBytes / (4 * row) / 32 * 32);
        const int S = (int)(row | 1);
        const size_t smem = (G - 1) * S * 4 + row * 4;
        B2S_TRY(smem_optin<deinterleave_kernel>(ctx, kMaxOuts * 2 * 32 * 4 + 32 * 4));
        const size_t grid = ceil_div(m, G);
        if (grid > 0x7FFFFFFFu) return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_fanout_exec: %zu groups in one call", m);
        deinterleave_kernel<<<(unsigned)grid, kThreads, smem, ctx->stream>>>((const float *)d_in, ptrs, (int)n_outs, w, m,
                                                                           (int)G, S);
    }
    B2S_CHECK_LAUNCH(ctx);
    *consumed = in_items;
    *produced = m;
    return B2S_OK;
}

}  // extern "C"
