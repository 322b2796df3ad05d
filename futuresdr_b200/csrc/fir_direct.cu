// fir_direct.cu -- CUDA-core direct-form FIR / decimating FIR for sm_90a.
//
// Computes the reference's   o[k] = sum_t i[D-1 + k*D + t] * taps[N-1-t]
// (crates/futuredsp/src/fir.rs:77-88 for D == 1, decimating_fir.rs:80-92 for D > 1) for the
// three sample/tap kinds futuredsp implements (fir.rs:206-276).
//
// Design (see DESIGN.md "direct FIR"):
//  * a CTA produces TK = THREADS*R consecutive outputs; it stages the D*(TK+Upad) input items
//    it needs in shared memory, DE-INTERLEAVED into D phase rows  x_q[m] = x[D*m + q], so the
//    decimator becomes D ordinary (stride-1) FIRs  o[k] = sum_q sum_u x_q[k+u] * G_q[u]
//    and the inner loop is identical for every D;
//  * each thread owns R consecutive outputs and slides an R+R-1 item register window over
//    its phase row: one 16-byte-vector segment load (R items) + R taps feed R*R MACs, so the
//    kernel is FMA-issue bound, not LDS bound;
//  * shared memory is XOR-swizzled at 16-byte granularity (chunk ^= (chunk>>3)&7) so the
//    R-item-strided segment loads of a quarter-warp hit 8 distinct bank groups;
//  * results are transposed through shared memory so global stores are fully coalesced
//    16-byte vectors; loads are float4-vectorised when D == 1.
// Accumulation is FP32 FMA; the summation order differs from the reference's strict
// left-to-right order (it is tap-order within a thread, but fused): parity is to 1e-5 relative
// (tests/test_gpu_fir.py).
#include "fir.cuh"

namespace {

__device__ __forceinline__ int swz(int chunk) { return chunk ^ ((chunk >> 3) & 7); }

using ::mac;   // complex sample x real tap (common.cuh)
__device__ __forceinline__ void mac(float &a, float x, float t) { a = fmaf(x, t, a); }
// Complex tap: accum + sample*tap, re = xr*tr - xi*ti, im = xr*ti + xi*tr (fir.rs:257-276)
__device__ __forceinline__ void mac(float2 &a, float2 x, float2 t) {
    a.x = fmaf(x.x, t.x, a.x);
    a.x = fmaf(-x.y, t.y, a.x);
    a.y = fmaf(x.x, t.y, a.y);
    a.y = fmaf(x.y, t.x, a.y);
}

template <typename S> __device__ __forceinline__ S zero_of();
template <> __device__ __forceinline__ float zero_of<float>() { return 0.0f; }
template <> __device__ __forceinline__ float2 zero_of<float2>() { return make_float2(0.f, 0.f); }

// rq: phase-row index; XOR-ing it into the chunk swizzle keeps a row's own reads conflict-free
// (a constant XOR permutes the 8 bank groups) and spreads the de-interleaving stores of the D
// phases -- which hit the same column of D different rows -- over different bank groups.
template <typename S, int R>
__device__ __forceinline__ void load_segment(S (&dst)[R], const unsigned char *row, int seg, int rq) {
    constexpr int EPC = 16 / sizeof(S);   // items per 16-byte chunk
    constexpr int CPS = R / EPC;          // chunks per R-item segment
#pragma unroll
    for (int j = 0; j < CPS; j++) {
        const int chunk = seg * CPS + j;
        const float4 v = *reinterpret_cast<const float4 *>(row + (swz(chunk) ^ rq) * 16);
        if constexpr (sizeof(S) == 8) {
            dst[2 * j] = *reinterpret_cast<const S *>(&v.x);
            dst[2 * j + 1] = *reinterpret_cast<const S *>(&v.z);
        } else {
            dst[4 * j] = *reinterpret_cast<const S *>(&v.x);
            dst[4 * j + 1] = *reinterpret_cast<const S *>(&v.y);
            dst[4 * j + 2] = *reinterpret_cast<const S *>(&v.z);
            dst[4 * j + 3] = *reinterpret_cast<const S *>(&v.w);
        }
    }
}

// R taps (warp-uniform) as 16-byte broadcast loads; g is 32-byte aligned
template <typename T, int R>
__device__ __forceinline__ void load_taps(T (&tp)[R], const T *g) {
    constexpr int NV = R * sizeof(T) / 16;
    const float4 *gv = reinterpret_cast<const float4 *>(g);
#pragma unroll
    for (int v = 0; v < NV; v++) reinterpret_cast<float4 *>(tp)[v] = gv[v];
}
// acc[r] += sum_j window[r + j] * tp[j] over the 2R-item window (lo | hi); all indices are static after
// unrolling, so sliding the window is a matter of swapping the roles of the two segment arrays in the
// caller -- no register moves (the first version copied hi -> lo after every chunk: 17 % of the loop).
template <typename S, typename T, int R>
__device__ __forceinline__ void mac_chunk(S (&acc)[R], const S (&lo)[R], const S (&hi)[R], const T (&tp)[R]) {
#pragma unroll
    for (int j = 0; j < R; j++) {
#pragma unroll
        for (int r = 0; r < R; r++) mac(acc[r], (r + j < R) ? lo[(r + j) % R] : hi[(r + j) % R], tp[j]);
    }
}
// one phase row: nchunk chunks of R taps against the thread's sliding window starting at segment seg0
template <typename S, typename T, int R>
__device__ __forceinline__ void fir_row(S (&acc)[R], const unsigned char *row, int rq, int seg0, const T *g, int nchunk) {
    S a[R], b[R];
    T tp[R];
    load_segment<S, R>(a, row, seg0, rq);
    int c = 0;
    for (; c + 1 < nchunk; c += 2) {
        load_segment<S, R>(b, row, seg0 + c + 1, rq);
        load_taps<T, R>(tp, g + c * R);
        mac_chunk<S, T, R>(acc, a, b, tp);
        load_segment<S, R>(a, row, seg0 + c + 2, rq);
        load_taps<T, R>(tp, g + (c + 1) * R);
        mac_chunk<S, T, R>(acc, b, a, tp);
    }
    if (c < nchunk) {
        load_segment<S, R>(b, row, seg0 + c + 1, rq);
        load_taps<T, R>(tp, g + c * R);
        mac_chunk<S, T, R>(acc, a, b, tp);
    }
}

// The same phase row against LT tap tables at once (the rational resampler's L polyphase banks, `bank_stride` floats
// apart): every window segment is loaded ONCE and multiplied into all LT accumulator sets, so the shared-memory
// traffic per MAC drops by LT (ncu on the one-bank-at-a-time loop: LSU wavefronts and the FMA pipe within 20 % of each other).
template <typename S, int R, int LT>
__device__ __forceinline__ void fir_row_banks(S (&acc)[LT][R], const unsigned char *row, int rq, int seg0, const float *g,
                                              int bank_stride, int nchunk) {
    S a[R], b[R];
    float tp[R];
    load_segment<S, R>(a, row, seg0, rq);
    int c = 0;
    for (; c + 1 < nchunk; c += 2) {
        load_segment<S, R>(b, row, seg0 + c + 1, rq);
#pragma unroll
        for (int k = 0; k < LT; k++) {
            load_taps<float, R>(tp, g + k * bank_stride + c * R);
            mac_chunk<S, float, R>(acc[k], a, b, tp);
        }
        load_segment<S, R>(a, row, seg0 + c + 2, rq);
#pragma unroll
        for (int k = 0; k < LT; k++) {
            load_taps<float, R>(tp, g + k * bank_stride + (c + 1) * R);
            mac_chunk<S, float, R>(acc[k], b, a, tp);
        }
    }
    if (c < nchunk) {
        load_segment<S, R>(b, row, seg0 + c + 1, rq);
#pragma unroll
        for (int k = 0; k < LT; k++) {
            load_taps<float, R>(tp, g + k * bank_stride + c * R);
            mac_chunk<S, float, R>(acc[k], a, b, tp);
        }
    }
}

// Interior-tile staging for D > 1: the tile's D*W items are all inside the input and the base is 16-byte
// aligned, so whole groups of THREADS*UNR float4 chunks are loaded with no predicates, 32-bit offsets and a
// running pointer; the ragged end of the tile and edge tiles go through the generic loops in the kernels.
// (ncu on the decimator: the generic loop was 42 % of all issued instructions, ~70 per float4.)
// Returns the number of chunks it staged; the caller finishes [ret, nchunks).
template <typename S, int THREADS>
__device__ __forceinline__ int stage_phases_interior(const S *__restrict__ in, long long s0, int D, int nchunks,
                                                     unsigned pitch_bytes, unsigned char *xs, int tid) {
    constexpr int EPC = 16 / sizeof(S);
    constexpr int UNR = 4;
    const int groups = nchunks / (THREADS * UNR);
    const float4 *p = reinterpret_cast<const float4 *>(in + s0) + tid;
    unsigned q = (unsigned)(tid * EPC) % (unsigned)D, m = (unsigned)(tid * EPC) / (unsigned)D;
    const unsigned dq = (unsigned)(THREADS * EPC) % (unsigned)D, dm = (unsigned)(THREADS * EPC) / (unsigned)D;
    for (int g = 0; g < groups; g++) {
        float4 v[UNR];
#pragma unroll
        for (int u = 0; u < UNR; u++) v[u] = __ldg(p + u * THREADS);
        p += UNR * THREADS;
#pragma unroll
        for (int u = 0; u < UNR; u++) {
            const S *items = reinterpret_cast<const S *>(&v[u]);
            unsigned qe = q, me = m;
#pragma unroll
            for (int e = 0; e < EPC; e++) {
                const unsigned ch = me / EPC;
                const unsigned sw = ch ^ ((ch >> 3) & 7u) ^ (qe & 7u);
                *reinterpret_cast<S *>(xs + qe * pitch_bytes + sw * 16u + (me % EPC) * (unsigned)sizeof(S)) = items[e];
                if (++qe == (unsigned)D) { qe = 0; ++me; }
            }
            q += dq; m += dm;
            if (q >= (unsigned)D) { q -= (unsigned)D; ++m; }
        }
    }
    return groups * THREADS * UNR;
}

// S: sample type (float | float2), T: tap type (float | float2)
template <typename S, typename T, int R, int THREADS>
__global__ void __launch_bounds__(THREADS)
fir_direct_kernel(const S *__restrict__ in, S *__restrict__ out, const T *__restrict__ ptaps,
                  int D, int Upad, int pitch /*items per phase row, multiple of 8 chunks*/,
                  long long n_in, long long n_out, int vec_ok) {
    constexpr int EPC = 16 / sizeof(S);
    constexpr int TK = THREADS * R;
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x;
    const long long k0 = (long long)blockIdx.x * TK;
    const int W = TK + Upad;                       // items needed per phase row
    unsigned char *xs = smem;                      // [D][pitch] items, swizzled per row
    T *gs = reinterpret_cast<T *>(smem + (size_t)D * pitch * sizeof(S));   // [D][Upad]

    // ---- stage taps
    for (int j = tid; j < D * Upad; j += THREADS) gs[j] = ptaps[j];

    // ---- stage inputs, de-interleaving phases
    const long long s0 = k0 * D;                   // first input item of this tile
    if (D == 1 && vec_ok) {
        const int nchunks = (W + EPC - 1) / EPC;
        for (int c = tid; c < nchunks; c += THREADS) {
            const long long s = s0 + (long long)c * EPC;
            float4 v;
            if (s + EPC <= n_in) {
                v = __ldg(reinterpret_cast<const float4 *>(in + s));
            } else {
                S tmp[EPC];
#pragma unroll
                for (int e = 0; e < EPC; e++) tmp[e] = (s + e < n_in) ? in[s + e] : zero_of<S>();
                v = *reinterpret_cast<float4 *>(tmp);
            }
            *reinterpret_cast<float4 *>(xs + swz(c) * 16) = v;
        }
    } else if (vec_ok) {
        // Decimator: 16-byte loads, four in flight per thread (the scalar loop below keeps too few bytes
        // in flight to cover HBM latency), then scatter the EPC items of
        // each chunk into their phase rows.  (q, m) of a thread's chunks advance by a fixed step, so
        // there is one integer division per thread, not per item.  s0 * sizeof(S) is a multiple of 16.
        const int total = D * W;
        const int nchunks = (total + EPC - 1) / EPC;
        constexpr int UNR = 4;
        int done = 0;                               // chunks already staged by the predicate-free path
        if (s0 + (long long)nchunks * EPC <= n_in)
            done = stage_phases_interior<S, THREADS>(in, s0, D, nchunks, (unsigned)(pitch * sizeof(S)), xs, tid);
        int q = (int)(((long long)done + tid) * EPC % D), m = (int)(((long long)done + tid) * EPC / D);
        const int dq = (THREADS * EPC) % D, dm = (THREADS * EPC) / D;
        for (int c0 = done + tid; c0 < nchunks; c0 += THREADS * UNR) {
            float4 v[UNR];
#pragma unroll
            for (int u = 0; u < UNR; u++) {
                const int c = c0 + u * THREADS;
                const long long s = s0 + (long long)c * EPC;
                if (c < nchunks && s + EPC <= n_in) {
                    v[u] = __ldg(reinterpret_cast<const float4 *>(in + s));
                } else {
                    S tmp[EPC];
#pragma unroll
                    for (int e = 0; e < EPC; e++) tmp[e] = (c < nchunks && s + e < n_in) ? in[s + e] : zero_of<S>();
                    v[u] = *reinterpret_cast<float4 *>(tmp);
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; u++) {
                const int c = c0 + u * THREADS;
                const S *items = reinterpret_cast<const S *>(&v[u]);
                int qe = q, me = m;
#pragma unroll
                for (int e = 0; e < EPC; e++) {
                    if (c < nchunks && c * EPC + e < total) {
                        const int chunk = me / EPC, el = me % EPC;
                        *reinterpret_cast<S *>(xs + ((size_t)qe * pitch + (swz(chunk) ^ (qe & 7)) * EPC + el) * sizeof(S)) = items[e];
                    }
                    if (++qe == D) { qe = 0; me++; }
                }
                q += dq; m += dm;
                if (q >= D) { q -= D; m += 1; }
            }
        }
    } else {
        // item j of the tile -> phase q = j % D, row index m = j / D (s0 is a multiple of D)
        const int total = D * W;
        int q = tid % D, m = tid / D;
        const int dq = THREADS % D, dm = THREADS / D;
        for (int j = tid; j < total; j += THREADS) {
            const long long s = s0 + j;
            const S v = (s < n_in) ? in[s] : zero_of<S>();
            const int chunk = m / EPC, e = m % EPC;
            *reinterpret_cast<S *>(xs + ((size_t)q * pitch + (swz(chunk) ^ (q & 7)) * EPC + e) * sizeof(S)) = v;
            q += dq; m += dm;
            if (q >= D) { q -= D; m += 1; }
        }
    }
    __syncthreads();

    // ---- R outputs per thread, sliding register window
    S acc[R];
#pragma unroll
    for (int r = 0; r < R; r++) acc[r] = zero_of<S>();

    const int nchunk_taps = Upad / R;
    for (int q = 0; q < D; q++)
        fir_row<S, T, R>(acc, xs + (size_t)q * pitch * sizeof(S), q & 7, tid, gs + q * Upad, nchunk_taps);
    __syncthreads();                                // everyone is done reading xs

    // ---- transpose through smem, coalesced vector stores
    {
        constexpr int CPS = R / EPC;
#pragma unroll
        for (int j = 0; j < CPS; j++) {
            const int chunk = tid * CPS + j;
            float4 v;
            if constexpr (sizeof(S) == 8) {
                v = make_float4(acc[2 * j].x, acc[2 * j].y, acc[2 * j + 1].x, acc[2 * j + 1].y);
            } else {
                v = make_float4(*reinterpret_cast<float *>(&acc[4 * j]),
                                *reinterpret_cast<float *>(&acc[4 * j + 1]),
                                *reinterpret_cast<float *>(&acc[4 * j + 2]),
                                *reinterpret_cast<float *>(&acc[4 * j + 3]));
            }
            *reinterpret_cast<float4 *>(xs + swz(chunk) * 16) = v;
        }
    }
    __syncthreads();
    {
        constexpr int NCH = TK / EPC;
        for (int c = tid; c < NCH; c += THREADS) {
            const long long k = k0 + (long long)c * EPC;
            if (k >= n_out) break;
            const float4 v = *reinterpret_cast<const float4 *>(xs + swz(c) * 16);
            if (vec_ok && k + EPC <= n_out) {
                *reinterpret_cast<float4 *>(out + k) = v;
            } else {
                const S *p = reinterpret_cast<const S *>(&v);
#pragma unroll
                for (int e = 0; e < EPC; e++)
                    if (k + e < n_out) out[k + e] = p[e];
            }
        }
    }
}

// Fallback for exotic shapes (very large decimation): one thread per output, straight from
// global memory (L1/L2 cached), reference tap order.
template <typename S, typename T>
__global__ void fir_naive_kernel(const S *__restrict__ in, S *__restrict__ out,
                                 const T *__restrict__ rtaps /* g[t] = taps[N-1-t] */, int N, int D,
                                 long long n_out) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_out) return;
    const S *x = in + (long long)D * k + (D - 1);
    S acc = zero_of<S>();
    for (int t = 0; t < N; t++) mac(acc, x[t], rtaps[t]);
    out[k] = acc;
}

// ---------------------------------------------------------------------------------------------
// Rational resampler on the same machinery (futuredsp::PolyphaseResamplingFir,
// polyphase_resampling_fir.rs:70-124):   o[k] = sum_t i[floor(k*M/L) + t] * taps[L*(T-1-t) + (k*M mod L)].
// Write k = L*j + k0: outputs with the same k0 share a polyphase bank and their windows start
// M items apart, i.e. for every k0 the resampler is a decimate-by-M FIR:
//      o[L*j + k0] = sum_q sum_u x_q[j + u] * G[k0][q][u],     x_q[m] = i[M*m + q]
// with G[k0][q][u] = bank_k0[M*u + q - s_k0], s_k0 = floor(k0*M/L) (host table, zero padded to a
// multiple of R).  A CTA stages the M phase rows of its input tile ONCE, then runs the sliding
// register-window loop of the direct FIR over the L banks -- for L = 2..4 (LT = L) every window segment is
// loaded once and multiplied into all L accumulator sets, otherwise (LT = 0) one pass per k0 -- and stages
// each thread's R*L outputs contiguously, in final order, in shared memory (segments R*L + 1 items apart)
// so that global stores are contiguous 16-byte vectors.  Compared with one thread per output reading every
// sample from shared memory (resamp.cu) this does LT*R*R MACs per R-item segment load instead of 1.6 FMA
// per LDS.
// ---------------------------------------------------------------------------------------------
template <typename S, int R, int THREADS, int LT>
__global__ void __launch_bounds__(THREADS, LT == 3 ? 5 : 1)        // L = 3: 99 -> 94 registers = a fifth resident CTA, no spills
resamp_slide_kernel(const S *__restrict__ in, S *__restrict__ out, const float *__restrict__ gtab,
                    int L, int M, int Upad, int pitch /*items per phase row*/, int opitch /*bytes of the output staging*/,
                    int os_off /*byte offset of the output staging: 0 = it reuses the input rows*/,
                    long long n_in, long long n_out, int vec_ok) {
    constexpr int EPC = 16 / sizeof(S);
    constexpr int TK = THREADS * R;                 // j's per CTA; the CTA produces L*TK outputs
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x;
    const long long j0 = (long long)blockIdx.x * TK;
    const int W = TK + Upad;
    unsigned char *xs = smem;                                                    // [M][pitch] items
    unsigned char *os = smem + os_off;                                           // THREADS segments of R*L + 1 items (opitch bytes in all)
    const size_t xs_bytes = (size_t)M * pitch * sizeof(S);
    float *gs = reinterpret_cast<float *>(smem + (os_off ? xs_bytes + opitch : (xs_bytes > (size_t)opitch ? xs_bytes : (size_t)opitch)));   // [L][M][Upad]

    for (int i = tid; i < L * M * Upad; i += THREADS) gs[i] = gtab[i];

    // ---- stage the input tile, de-interleaved into M phase rows (same scheme as the decimator)
    const long long s0 = j0 * M;
    const int total = M * W;
    if (vec_ok) {
        const int nchunks = (total + EPC - 1) / EPC;
        constexpr int UNR = 4;
        int done = 0;
        if (s0 + (long long)nchunks * EPC <= n_in)
            done = stage_phases_interior<S, THREADS>(in, s0, M, nchunks, (unsigned)(pitch * sizeof(S)), xs, tid);
        int q = (int)(((long long)done + tid) * EPC % M), m = (int)(((long long)done + tid) * EPC / M);
        const int dq = (THREADS * EPC) % M, dm = (THREADS * EPC) / M;
        for (int c0 = done + tid; c0 < nchunks; c0 += THREADS * UNR) {
            float4 v[UNR];
#pragma unroll
            for (int u = 0; u < UNR; u++) {
                const int c = c0 + u * THREADS;
                const long long s = s0 + (long long)c * EPC;
                if (c < nchunks && s + EPC <= n_in) {
                    v[u] = __ldg(reinterpret_cast<const float4 *>(in + s));
                } else {
                    S tmp[EPC];
#pragma unroll
                    for (int e = 0; e < EPC; e++) tmp[e] = (c < nchunks && s + e < n_in) ? in[s + e] : zero_of<S>();
                    v[u] = *reinterpret_cast<float4 *>(tmp);
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; u++) {
                const int c = c0 + u * THREADS;
                const S *items = reinterpret_cast<const S *>(&v[u]);
                int qe = q, me = m;
#pragma unroll
                for (int e = 0; e < EPC; e++) {
                    if (c < nchunks && c * EPC + e < total) {
                        const int chunk = me / EPC, el = me % EPC;
                        *reinterpret_cast<S *>(xs + ((size_t)qe * pitch + (swz(chunk) ^ (qe & 7)) * EPC + el) * sizeof(S)) = items[e];
                    }
                    if (++qe == M) { qe = 0; me++; }
                }
                q += dq; m += dm;
                if (q >= M) { q -= M; m += 1; }
            }
        }
    } else {
        int q = tid % M, m = tid / M;
        const int dq = THREADS % M, dm = THREADS / M;
        for (int j = tid; j < total; j += THREADS) {
            const long long s = s0 + j;
            const S v = (s < n_in) ? in[s] : zero_of<S>();
            const int chunk = m / EPC, e = m % EPC;
            *reinterpret_cast<S *>(xs + ((size_t)q * pitch + (swz(chunk) ^ (q & 7)) * EPC + e) * sizeof(S)) = v;
            q += dq; m += dm;
            if (q >= M) { q -= M; m += 1; }
        }
    }
    __syncthreads();

    // ---- one sliding-window pass per k0
    const int nchunk_taps = Upad / R;
    if constexpr (LT > 0) {
        S acc[LT][R];
#pragma unroll
        for (int k = 0; k < LT; k++)
#pragma unroll
            for (int r = 0; r < R; r++) acc[k][r] = zero_of<S>();
        for (int q = 0; q < M; q++)
            fir_row_banks<S, R, LT>(acc, xs + (size_t)q * pitch * sizeof(S), q & 7, tid, gs + (size_t)q * Upad, M * Upad, nchunk_taps);
        if (os_off == 0) __syncthreads();                // the staging reuses the input rows: everyone is done reading them
        S *oseg = reinterpret_cast<S *>(os) + (size_t)tid * (R * LT + 1);
#pragma unroll
        for (int r = 0; r < R; r++)
#pragma unroll
            for (int k = 0; k < LT; k++) oseg[r * LT + k] = acc[k][r];
    } else {
        for (int k0 = 0; k0 < L; k0++) {
            S acc[R];
#pragma unroll
            for (int r = 0; r < R; r++) acc[r] = zero_of<S>();
            for (int q = 0; q < M; q++)
                fir_row<S, float, R>(acc, xs + (size_t)q * pitch * sizeof(S), q & 7, tid, gs + ((size_t)k0 * M + q) * Upad,
                                     nchunk_taps);
            // output staging in FINAL order: this thread's R*L outputs o = L*(R*tid + r) + k0 form one segment of R*L items;
            // segments are R*L + 1 items apart (odd stride: the lanes of a warp hit distinct banks)
            S *oseg = reinterpret_cast<S *>(os) + (size_t)tid * (R * L + 1) + k0;
#pragma unroll
            for (int r = 0; r < R; r++) oseg[r * L] = acc[r];
        }
    }
    __syncthreads();

    // ---- contiguous 16-byte vector stores; chunk c holds outputs [c*EPC, (c+1)*EPC) of the tile, which sit in ONE
    //      segment (R*L is a multiple of EPC) at item index p + p / (R*L)
    {
        const long long o0 = j0 * L;
        const int SEGL = R * L;
        const int nout_chunks = L * TK / EPC;                       // TK is a multiple of EPC
        const S *ob = reinterpret_cast<const S *>(os);
        int seg = (tid * EPC) / SEGL, rem = (tid * EPC) % SEGL;
        const int dseg = (THREADS * EPC) / SEGL, drem = (THREADS * EPC) % SEGL;
        for (int c = tid; c < nout_chunks; c += THREADS) {
            const long long o = o0 + (long long)c * EPC;
            if (o >= n_out) break;
            const S *src = ob + c * EPC + seg;
            S items[EPC];
#pragma unroll
            for (int e = 0; e < EPC; e++) items[e] = src[e];
            if (vec_ok && o + EPC <= n_out) {
                *reinterpret_cast<float4 *>(out + o) = *reinterpret_cast<float4 *>(items);
            } else {
#pragma unroll
                for (int e = 0; e < EPC; e++)
                    if (o + e < n_out) out[o + e] = items[e];
            }
            seg += dseg; rem += drem;
            if (rem >= SEGL) { rem -= SEGL; seg += 1; }
        }
    }
}

constexpr int kThreads = 128;
constexpr int kR = 8;
constexpr size_t kSmemBudget = 160 * 1024;

template <typename S, typename T>
int32_t launch_typed(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out,
                     cudaStream_t stream) {
    b2s_ctx *ctx = f->ctx;
    constexpr int EPC = 16 / sizeof(S);
    constexpr int TK = kThreads * kR;
    const int D = (int)f->decim;
    const int W = TK + f->Upad;
    const int pitch = (int)round_up((size_t)W, 8 * EPC);
    const size_t smem = (size_t)D * pitch * sizeof(S) + (size_t)D * f->Upad * sizeof(T);
    if (smem > kSmemBudget) {
        // taps for the naive kernel: phase table row-major does not apply; use d_ptaps tail
        const T *rt = reinterpret_cast<const T *>(f->d_ptaps) + (size_t)D * f->Upad;
        const int th = 256;
        fir_naive_kernel<S, T><<<(unsigned)ceil_div(n_out, th), th, 0, stream>>>(
            (const S *)d_in, (S *)d_out, rt, (int)f->ntaps, D, (long long)n_out);
        B2S_CHECK_LAUNCH(ctx);
        return B2S_OK;
    }
    auto kern = fir_direct_kernel<S, T, kR, kThreads>;
    static PerDeviceOnce optin;                  // per template instantiation, per device
    if (optin.need(ctx->device)) {
        B2S_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)kSmemBudget));
        optin.done(ctx->device);
    }
    const int vec_ok = ((reinterpret_cast<uintptr_t>(d_in) | reinterpret_cast<uintptr_t>(d_out)) & 15) == 0;
    const unsigned grid = (unsigned)ceil_div(n_out, (size_t)TK);
    kern<<<grid, kThreads, smem, stream>>>((const S *)d_in, (S *)d_out, (const T *)f->d_ptaps, D,
                                           f->Upad, pitch, (long long)n_in, (long long)n_out, vec_ok);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

}  // namespace

// Build G[q][u] (phase-major, reversed, zero padded to a multiple of R) followed by the plain
// reversed taps g[t] (used by the naive fallback).
int32_t fir_direct_prepare(b2s_fir *f) {
    b2s_ctx *ctx = f->ctx;
    const size_t N = f->ntaps, D = f->decim, tf = kind_tap_floats(f->kind);
    f->U = (int)((N + D - 2) / D + 1);
    f->Upad = (int)round_up((size_t)f->U, kR);
    std::vector<float> h((D * f->Upad + N) * tf, 0.0f);
    for (size_t q = 0; q < D; q++)
        for (size_t u = 0; u < (size_t)f->U; u++) {
            const long long idx = (long long)(D * u + q) - (long long)(D - 1);
            if (idx < 0 || idx >= (long long)N) continue;
            for (size_t c = 0; c < tf; c++)
                h[(q * f->Upad + u) * tf + c] = f->taps_host[(N - 1 - idx) * tf + c];
        }
    for (size_t t = 0; t < N; t++)
        for (size_t c = 0; c < tf; c++) h[(D * f->Upad + t) * tf + c] = f->taps_host[(N - 1 - t) * tf + c];
    B2S_CUDA(ctx, cudaMalloc((void **)&f->d_ptaps, h.size() * sizeof(float)));
    B2S_CUDA(ctx, cudaMemcpyAsync(f->d_ptaps, h.data(), h.size() * sizeof(float),
                                  cudaMemcpyHostToDevice, ctx->stream));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // h goes out of scope
    return B2S_OK;
}

int32_t fir_direct_launch(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out,
                          cudaStream_t stream) {
    if (n_out == 0) return B2S_OK;
    switch (f->kind) {
        case B2S_F32_F32: return launch_typed<float, float>(f, d_in, n_in, d_out, n_out, stream);
        case B2S_C32_F32: return launch_typed<float2, float>(f, d_in, n_in, d_out, n_out, stream);
        case B2S_C32_C32: return launch_typed<float2, float2>(f, d_in, n_in, d_out, n_out, stream);
    }
    return b2s_fail(f->ctx, B2S_EINVAL, "bad kind");
}

// ---- resampler entry points (used by resamp.cu) ------------------------------------------------
namespace {
constexpr int kRsSlideThreads = 128;
constexpr size_t kRsSlideSmemMax = 96 * 1024;        // keep >= 2 CTAs per SM
size_t resamp_slide_ostage(size_t L, size_t isz) { return round_up((size_t)kRsSlideThreads * (kR * L + 1) * isz, 16); }
bool resamp_slide_banks(size_t L) {                    // L with an all-banks-per-segment instantiation (resamp_slide_launch)
    static const bool off = getenv("B2S_RESAMP_NO_BANKS") != nullptr;         // A/B switch: one bank at a time
    return !off && L >= 2 && L <= 4;
}
size_t resamp_slide_smem(size_t L, size_t M, size_t Upad, size_t isz) {
    const size_t TK = (size_t)kRsSlideThreads * kR, EPC = 16 / isz;
    const size_t pitch = round_up(TK + Upad, 8 * EPC);
    const size_t xs = M * pitch * isz, os = resamp_slide_ostage(L, isz);
    // the all-banks kernel writes its outputs after the last read of the input rows, so the two stagings share memory
    return (resamp_slide_banks(L) ? std::max(xs, os) : xs + os) + L * M * Upad * sizeof(float);
}
}  // namespace

int resamp_slide_upad(size_t M, size_t T) { return (int)round_up((T + M - 2) / M + 1, (size_t)kR); }

bool resamp_slide_supported(size_t L, size_t M, size_t T, size_t item_bytes) {
    const size_t Upad = (size_t)resamp_slide_upad(M, T);
    // worthwhile only while the zero padding of the per-phase taps stays small (T/M taps per phase row)
    if (Upad * M > 2 * (T + M) + 16) return false;
    return resamp_slide_smem(L, M, Upad, item_bytes) <= kRsSlideSmemMax;
}

// G[k0][q][u] = bank_k0[M*u + q - s_k0],  bank_k0[t] = taps[L*(T-1-t) + (k0*M mod L)],  s_k0 = floor(k0*M/L)
void resamp_slide_table(const float *taps, size_t L, size_t M, size_t T, std::vector<float> &g) {
    const size_t Upad = (size_t)resamp_slide_upad(M, T);
    g.assign(L * M * Upad, 0.0f);
    for (size_t k0 = 0; k0 < L; k0++) {
        const size_t bank = (k0 * M) % L, s = (k0 * M) / L;
        for (size_t q = 0; q < M; q++)
            for (size_t u = 0; u < Upad; u++) {
                const long long t = (long long)(M * u + q) - (long long)s;
                if (t < 0 || t >= (long long)T) continue;
                g[(k0 * M + q) * Upad + u] = taps[L * (T - 1 - (size_t)t) + bank];
            }
    }
}

int32_t resamp_slide_launch(b2s_ctx *ctx, b2s_kind kind, const float *d_gtab, size_t L, size_t M, size_t T,
                            const void *d_in, size_t n_in, void *d_out, size_t n_out, cudaStream_t stream) {
    const size_t isz = kind_in_bytes(kind), EPC = 16 / isz;
    const size_t Upad = (size_t)resamp_slide_upad(M, T);
    const size_t TK = (size_t)kRsSlideThreads * kR;
    const int pitch = (int)round_up(TK + Upad, 8 * EPC), opitch = (int)resamp_slide_ostage(L, isz);
    const size_t smem = resamp_slide_smem(L, M, Upad, isz);
    const int os_off = resamp_slide_banks(L) ? 0 : (int)((size_t)M * pitch * isz);
    const int vec_ok = ((reinterpret_cast<uintptr_t>(d_in) | reinterpret_cast<uintptr_t>(d_out)) & 15) == 0;
    const unsigned grid = (unsigned)ceil_div(n_out, L * TK);
#define RS_SLIDE(S, LT)                                                                                                    \
    do {                                                                                                                   \
        auto kern = resamp_slide_kernel<S, kR, kRsSlideThreads, LT>;                                                       \
        static PerDeviceOnce optin;                                                                                        \
        if (optin.need(ctx->device)) {                                                                                     \
            B2S_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRsSlideSmemMax));  \
            optin.done(ctx->device);                                                                                       \
        }                                                                                                                  \
        kern<<<grid, kRsSlideThreads, smem, stream>>>((const S *)d_in, (S *)d_out, d_gtab, (int)L, (int)M, (int)Upad,      \
                                                      pitch, opitch, os_off, (long long)n_in, (long long)n_out, vec_ok);   \
    } while (0)
    const size_t lt = resamp_slide_banks(L) ? L : 0;
    if (kind == B2S_F32_F32) {
        if (lt == 2) RS_SLIDE(float, 2); else if (lt == 3) RS_SLIDE(float, 3); else if (lt == 4) RS_SLIDE(float, 4); else RS_SLIDE(float, 0);
    } else {
        if (lt == 2) RS_SLIDE(float2, 2); else if (lt == 3) RS_SLIDE(float2, 3); else if (lt == 4) RS_SLIDE(float2, 4); else RS_SLIDE(float2, 0);
    }
#undef RS_SLIDE
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}
