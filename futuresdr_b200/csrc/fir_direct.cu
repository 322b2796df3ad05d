// fir_direct.cu -- CUDA-core sliding-window kernel for sm_90a: the direct-form FIR, the decimating FIR and the
// rational resampler for small L*M.
//
// The FIR computes the reference's   o[k] = sum_t i[D-1 + k*D + t] * taps[N-1-t]
// (crates/futuredsp/src/fir.rs:77-88 for D == 1, decimating_fir.rs:80-92 for D > 1) for the three sample/tap kinds
// futuredsp implements (fir.rs:206-276); the resampler (futuredsp::PolyphaseResamplingFir,
// polyphase_resampling_fir.rs:70-124) computes   o[k] = sum_t i[floor(k*M/L) + t] * taps[L*(T-1-t) + (k*M mod L)].
// Write k = L*j + k0: outputs with the same k0 share the polyphase bank bank_k0[t] = taps[L*(T-1-t) + (k0*M mod L)]
// and their windows start M items apart, so for every k0 the resampler is a decimate-by-M FIR:
//      o[L*j + k0] = sum_q sum_u x_q[j + u] * G[k0][q][u],     x_q[m] = i[M*m + q],
//      G[k0][q][u] = bank_k0[M*u + q - s_k0],  s_k0 = floor(k0*M/L)      (host table, zero padded to a multiple of R)
// The FIR is the case L = 1, M = D, bank_0[t] = taps[N-1-t] with the shift s_0 = D-1, and one kernel runs both.
//
// Design (see DESIGN.md "direct FIR"):
//  * a CTA produces the outputs of TK = THREADS*R consecutive j; it stages the M*(TK+Upad) input items they
//    need in shared memory, DE-INTERLEAVED into M phase rows x_q, so the inner loop is a stride-1 FIR for every M;
//  * each thread owns R consecutive j and slides an R+R-1 item register window over each phase row: one
//    16-byte-vector segment load (R items) + R taps feed R*R MACs per bank, so the kernel is FMA-issue bound, not
//    LDS bound; for L = 2..4 every segment is multiplied into all L banks, for L >= 5 there is one pass per bank;
//  * shared memory is XOR-swizzled at 16-byte granularity (chunk ^= (chunk>>3)&7) so the
//    R-item-strided segment loads of a quarter-warp hit 8 distinct bank groups;
//  * results go through shared memory so global stores are contiguous 16-byte vectors: a swizzled transpose for
//    L = 1, each thread's R*L outputs in final order for L > 1; loads are float4-vectorised.
// Accumulation is FP32 FMA; the summation order differs from the reference's strict
// left-to-right order (it is tap-order within a phase row, but fused): parity is to 1e-5 relative
// (tests/test_gpu_fir.py, tests/test_gpu_blocks.py).
#include "fir.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kR = 8;
constexpr int kTK = kThreads * kR;
constexpr int kMaxBanks = 4;                  // L up to this: all banks per segment load, output staging reuses the input rows
constexpr size_t kSmemMax = 160 * 1024;      // the FIR's tile budget (fir_naive_kernel above it)
constexpr size_t kRsSmemMax = 96 * 1024;     // the resampler's: keep >= 2 CTAs per SM (resamp_kernel above it)

__device__ __forceinline__ int swz(int chunk) { return chunk ^ ((chunk >> 3) & 7); }

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

// One phase row: nchunk chunks of R taps against the thread's sliding window starting at segment seg0, for LT tap
// tables `bank_stride` taps apart (the resampler's polyphase banks): every window segment is loaded ONCE and multiplied
// into all LT accumulator sets, so the shared-memory traffic per MAC drops by LT (ncu on the one-bank-at-a-time loop:
// LSU wavefronts and the FMA pipe within 20 % of each other).
template <typename S, typename T, int R, int LT>
__device__ __forceinline__ void fir_row_banks(S (&acc)[LT][R], const unsigned char *row, int rq, int seg0, const T *g,
                                              int bank_stride, int nchunk) {
    S a[R], b[R];
    T tp[R];
    load_segment<S, R>(a, row, seg0, rq);
    int c = 0;
    for (; c + 1 < nchunk; c += 2) {
        load_segment<S, R>(b, row, seg0 + c + 1, rq);
#pragma unroll
        for (int k = 0; k < LT; k++) {
            load_taps<T, R>(tp, g + k * bank_stride + c * R);
            mac_chunk<S, T, R>(acc[k], a, b, tp);
        }
        load_segment<S, R>(a, row, seg0 + c + 2, rq);
#pragma unroll
        for (int k = 0; k < LT; k++) {
            load_taps<T, R>(tp, g + k * bank_stride + (c + 1) * R);
            mac_chunk<S, T, R>(acc[k], b, a, tp);
        }
    }
    if (c < nchunk) {
        load_segment<S, R>(b, row, seg0 + c + 1, rq);
#pragma unroll
        for (int k = 0; k < LT; k++) {
            load_taps<T, R>(tp, g + k * bank_stride + c * R);
            mac_chunk<S, T, R>(acc[k], a, b, tp);
        }
    }
}

// Interior-tile staging for M > 1: the tile's M*W items are all inside the input and the base is 16-byte
// aligned, so whole groups of THREADS*UNR float4 chunks are loaded with no predicates, 32-bit offsets and a
// running pointer; the ragged end of the tile and edge tiles go through the generic loop in stage_phases.
// (ncu on the decimator: the generic loop was 42 % of all issued instructions, ~70 per float4.)
// Returns the number of chunks it staged; the caller finishes [ret, nchunks).
template <typename S>
__device__ __forceinline__ int stage_phases_interior(const S *__restrict__ in, long long s0, int M, int nchunks,
                                                     unsigned pitch_bytes, unsigned char *xs, int tid) {
    constexpr int EPC = 16 / sizeof(S);
    constexpr int UNR = 4;
    const int groups = nchunks / (kThreads * UNR);
    const float4 *p = reinterpret_cast<const float4 *>(in + s0) + tid;
    unsigned q = (unsigned)(tid * EPC) % (unsigned)M, m = (unsigned)(tid * EPC) / (unsigned)M;
    const unsigned dq = (unsigned)(kThreads * EPC) % (unsigned)M, dm = (unsigned)(kThreads * EPC) / (unsigned)M;
    for (int g = 0; g < groups; g++) {
        float4 v[UNR];
#pragma unroll
        for (int u = 0; u < UNR; u++) v[u] = __ldg(p + u * kThreads);
        p += UNR * kThreads;
#pragma unroll
        for (int u = 0; u < UNR; u++) {
            const S *items = reinterpret_cast<const S *>(&v[u]);
            unsigned qe = q, me = m;
#pragma unroll
            for (int e = 0; e < EPC; e++) {
                const unsigned ch = me / EPC;
                const unsigned sw = ch ^ ((ch >> 3) & 7u) ^ (qe & 7u);
                *reinterpret_cast<S *>(xs + qe * pitch_bytes + sw * 16u + (me % EPC) * (unsigned)sizeof(S)) = items[e];
                if (++qe == (unsigned)M) { qe = 0; ++me; }
            }
            q += dq; m += dm;
            if (q >= (unsigned)M) { q -= (unsigned)M; ++m; }
        }
    }
    return groups * kThreads * UNR;
}

// Stages the tile's M*W input items from s0 (a multiple of M) on, zero past n_in, de-interleaved into the M phase rows
// x_q[m] = in[s0 + M*m + q] of `pitch` items each.  vec_ok: `in` is 16-byte aligned (s0 * sizeof(S) always is).
// COPY1: M == 1 is a plain float4 copy.  Only the one-bank tile uses it: the resampler's M == 1 tiles (2/1, 5/1) keep the
// four loads in flight per thread of the loop below, which hide HBM latency better at their lower occupancy
// (5/1 c32 is 2.4 % faster that way on an H100 80GB HBM3 at 400 W).
template <typename S, bool COPY1>
__device__ __forceinline__ void stage_phases(const S *__restrict__ in, long long s0, int M, int W, int pitch,
                                             long long n_in, int vec_ok, unsigned char *xs, int tid) {
    constexpr int EPC = 16 / sizeof(S);
    if (COPY1 && M == 1 && vec_ok) {
        const int nchunks = (W + EPC - 1) / EPC;
        for (int c = tid; c < nchunks; c += kThreads) {
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
        // 16-byte loads, four in flight per thread (the scalar loop below keeps too few bytes
        // in flight to cover HBM latency), then scatter the EPC items of
        // each chunk into their phase rows.  (q, m) of a thread's chunks advance by a fixed step, so
        // there is one integer division per thread, not per item.
        const int total = M * W;
        const int nchunks = (total + EPC - 1) / EPC;
        constexpr int UNR = 4;
        int done = 0;                               // chunks already staged by the predicate-free path
        if (s0 + (long long)nchunks * EPC <= n_in)
            done = stage_phases_interior<S>(in, s0, M, nchunks, (unsigned)(pitch * sizeof(S)), xs, tid);
        int q = (int)(((long long)done + tid) * EPC % M), m = (int)(((long long)done + tid) * EPC / M);
        const int dq = (kThreads * EPC) % M, dm = (kThreads * EPC) / M;
        for (int c0 = done + tid; c0 < nchunks; c0 += kThreads * UNR) {
            float4 v[UNR];
#pragma unroll
            for (int u = 0; u < UNR; u++) {
                const int c = c0 + u * kThreads;
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
                const int c = c0 + u * kThreads;
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
        // item j of the tile -> phase q = j % M, row index m = j / M
        const int total = M * W;
        int q = tid % M, m = tid / M;
        const int dq = kThreads % M, dm = kThreads / M;
        for (int j = tid; j < total; j += kThreads) {
            const long long s = s0 + j;
            const S v = (s < n_in) ? in[s] : zero_of<S>();
            const int chunk = m / EPC, e = m % EPC;
            *reinterpret_cast<S *>(xs + ((size_t)q * pitch + (swz(chunk) ^ (q & 7)) * EPC + e) * sizeof(S)) = v;
            q += dq; m += dm;
            if (q >= M) { q -= M; m += 1; }
        }
    }
}

// S: sample type (float | float2), T: tap type (float | float2; float2 only with L = 1).
// LT: banks per pass -- 1 for L = 1, L for L = 2..kMaxBanks, 0 for a run-time loop over L > kMaxBanks banks.
// The CTA produces outputs [L*j0, L*(j0 + TK)).  Shared memory (slide_layout): [M][pitch] phase rows, the output
// staging (in the phase rows for LT > 0, right behind them for LT = 0), the [L][M][Upad] tap table at gs_off (right
// behind the phase rows for LT = 1).
// Minimum resident CTAs: LT = 3 asks for a fifth, which caps the float2 instantiation at 96 registers (ptxas, sm_90a,
// CUDA 12.9; no spills).  LT = 1 states none (0): with a minimum of 1 ptxas gives the FIR 56-59 registers instead of 48.
// L and gs_off come last: placed before n_in they change ptxas's schedule of the FIR, which made the f32 decimator
// 3 % slower at D = 16..25 (H100 80GB HBM3, 700 W).
template <typename S, typename T, int LT>
__global__ void __launch_bounds__(kThreads, LT == 3 ? 5 : LT == 1 ? 0 : 1)
fir_direct_kernel(const S *__restrict__ in, S *__restrict__ out, const T *__restrict__ gtab, int M, int Upad,
                  int pitch /*items per phase row, multiple of 8 chunks*/,
                  long long n_in, long long n_out, int vec_ok, int L, int gs_off) {
    constexpr int EPC = 16 / sizeof(S);
    constexpr int NB = LT > 0 ? LT : 1;             // banks per sliding-window pass
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x;
    const long long j0 = (long long)blockIdx.x * kTK;
    const size_t xs_bytes = (size_t)M * pitch * sizeof(S);
    unsigned char *xs = smem;
    unsigned char *os = smem + (LT == 0 ? xs_bytes : 0);
    T *gs = reinterpret_cast<T *>(smem + (LT == 1 ? xs_bytes : (size_t)gs_off));

    for (int i = tid; i < (LT > 0 ? LT : L) * M * Upad; i += kThreads) gs[i] = gtab[i];
    stage_phases<S, LT == 1>(in, j0 * M, M, kTK + Upad, pitch, n_in, vec_ok, xs, tid);
    __syncthreads();

    // ---- R j's per thread, sliding register window: all banks in one pass (LT > 0) or one pass per bank (LT = 0)
    const int nchunk_taps = Upad / kR;
    for (int k0 = 0; k0 < (LT > 0 ? 1 : L); k0++) {
        S acc[NB][kR];
#pragma unroll
        for (int k = 0; k < NB; k++)
#pragma unroll
            for (int r = 0; r < kR; r++) acc[k][r] = zero_of<S>();
        for (int q = 0; q < M; q++)
            fir_row_banks<S, T, kR, NB>(acc, xs + (size_t)q * pitch * sizeof(S), q & 7, tid,
                                        gs + (k0 * M + q) * Upad, M * Upad, nchunk_taps);
        if constexpr (LT == 0) {
            // output staging of its own, in FINAL order: this thread's R*L outputs o = L*(R*tid + r) + k0 form one
            // segment of R*L items; segments are R*L + 1 items apart (odd stride: the lanes of a warp hit distinct banks)
            S *oseg = reinterpret_cast<S *>(os) + (size_t)tid * (kR * L + 1) + k0;
#pragma unroll
            for (int r = 0; r < kR; r++) oseg[r * L] = acc[0][r];
        } else if constexpr (LT == 1) {
            __syncthreads();                        // the staging reuses the phase rows: everyone is done reading them
            constexpr int CPS = kR / EPC;
#pragma unroll
            for (int j = 0; j < CPS; j++) {
                const int chunk = tid * CPS + j;
                float4 v;
                if constexpr (sizeof(S) == 8) {
                    v = make_float4(acc[0][2 * j].x, acc[0][2 * j].y, acc[0][2 * j + 1].x, acc[0][2 * j + 1].y);
                } else {
                    v = make_float4(*reinterpret_cast<float *>(&acc[0][4 * j]),
                                    *reinterpret_cast<float *>(&acc[0][4 * j + 1]),
                                    *reinterpret_cast<float *>(&acc[0][4 * j + 2]),
                                    *reinterpret_cast<float *>(&acc[0][4 * j + 3]));
                }
                *reinterpret_cast<float4 *>(os + swz(chunk) * 16) = v;
            }
        } else {
            __syncthreads();                        // the staging reuses the phase rows: everyone is done reading them
            S *oseg = reinterpret_cast<S *>(os) + (size_t)tid * (kR * LT + 1);
#pragma unroll
            for (int r = 0; r < kR; r++)
#pragma unroll
                for (int k = 0; k < LT; k++) oseg[r * LT + k] = acc[k][r];
        }
    }
    __syncthreads();

    // ---- contiguous 16-byte vector stores
    if constexpr (LT == 1) {
        constexpr int NCH = kTK / EPC;
        for (int c = tid; c < NCH; c += kThreads) {
            const long long k = j0 + (long long)c * EPC;
            if (k >= n_out) break;
            const float4 v = *reinterpret_cast<const float4 *>(os + swz(c) * 16);
            if (vec_ok && k + EPC <= n_out) {
                *reinterpret_cast<float4 *>(out + k) = v;
            } else {
                const S *p = reinterpret_cast<const S *>(&v);
#pragma unroll
                for (int e = 0; e < EPC; e++)
                    if (k + e < n_out) out[k + e] = p[e];
            }
        }
    } else {
        // chunk c holds outputs [c*EPC, (c+1)*EPC) of the tile, which sit in ONE segment (R*L is a multiple of EPC)
        // at item index p + p / (R*L)
        const long long o0 = j0 * L;
        const int SEGL = kR * L;
        const int nout_chunks = L * kTK / EPC;
        const S *ob = reinterpret_cast<const S *>(os);
        int seg = (tid * EPC) / SEGL, rem = (tid * EPC) % SEGL;
        const int dseg = (kThreads * EPC) / SEGL, drem = (kThreads * EPC) % SEGL;
        for (int c = tid; c < nout_chunks; c += kThreads) {
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

// taps per phase row of the table, zero padded to a multiple of R: the index M*u + q - s of G stays below T for
// u < U whatever the shift s <= M-1
int slide_upad(size_t M, size_t T) { return (int)round_up((T + M - 2) / M + 1, (size_t)kR); }

struct SlideLayout {
    int pitch;                                  // items per phase row
    size_t gs_off, smem;                        // byte offset of the tap table; total bytes
};
SlideLayout slide_layout(size_t L, size_t M, size_t Upad, size_t isz, size_t tsz) {
    SlideLayout s;
    s.pitch = (int)round_up(kTK + Upad, 8 * (16 / isz));
    const size_t xs = M * s.pitch * isz;
    const size_t os = L == 1 ? kTK * isz : round_up(kThreads * (kR * L + 1) * isz, 16);
    // up to kMaxBanks banks the kernel writes its outputs after the last read of the phase rows, so the two share memory
    s.gs_off = L <= kMaxBanks ? std::max(xs, os) : xs + os;
    s.smem = s.gs_off + L * M * Upad * tsz;
    return s;
}

template <typename S, typename T, int LT>
int32_t slide_launch(b2s_ctx *ctx, const T *d_tab, int L, int M, int Upad, const SlideLayout &lay, const void *d_in,
                     size_t n_in, void *d_out, size_t n_out, cudaStream_t stream) {
    constexpr auto kern = fir_direct_kernel<S, T, LT>;
    B2S_TRY(smem_optin<kern>(ctx, kSmemMax));
    const int vec_ok = ((reinterpret_cast<uintptr_t>(d_in) | reinterpret_cast<uintptr_t>(d_out)) & 15) == 0;
    const unsigned grid = (unsigned)ceil_div(n_out, (size_t)L * kTK);
    kern<<<grid, kThreads, lay.smem, stream>>>((const S *)d_in, (S *)d_out, d_tab, M, Upad, lay.pitch,
                                               (long long)n_in, (long long)n_out, vec_ok, L, (int)lay.gs_off);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

template <typename S, typename T>
int32_t launch_typed(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out, cudaStream_t stream) {
    const int D = (int)f->decim;
    const SlideLayout lay = slide_layout(1, D, f->Upad, sizeof(S), sizeof(T));
    if (lay.smem > kSmemMax) {
        // the naive kernel reads the plain reversed taps behind the phase table
        const T *rt = reinterpret_cast<const T *>(f->d_ptaps.get()) + (size_t)D * f->Upad;
        const int th = 256;
        fir_naive_kernel<S, T><<<(unsigned)ceil_div(n_out, th), th, 0, stream>>>(
            (const S *)d_in, (S *)d_out, rt, (int)f->ntaps, D, (long long)n_out);
        B2S_CHECK_LAUNCH(f->ctx);
        return B2S_OK;
    }
    return slide_launch<S, T, 1>(f->ctx, reinterpret_cast<const T *>(f->d_ptaps.get()), 1, D, f->Upad, lay, d_in, n_in, d_out,
                                 n_out, stream);
}

template <typename S>
int32_t resamp_launch_typed(b2s_ctx *ctx, const float *d_gtab, int L, int M, int Upad, const void *d_in, size_t n_in,
                            void *d_out, size_t n_out, cudaStream_t stream) {
    const SlideLayout lay = slide_layout(L, M, Upad, sizeof(S), sizeof(float));
    switch (L) {
        case 1: return slide_launch<S, float, 1>(ctx, d_gtab, L, M, Upad, lay, d_in, n_in, d_out, n_out, stream);
        case 2: return slide_launch<S, float, 2>(ctx, d_gtab, L, M, Upad, lay, d_in, n_in, d_out, n_out, stream);
        case 3: return slide_launch<S, float, 3>(ctx, d_gtab, L, M, Upad, lay, d_in, n_in, d_out, n_out, stream);
        case 4: return slide_launch<S, float, 4>(ctx, d_gtab, L, M, Upad, lay, d_in, n_in, d_out, n_out, stream);
        default: return slide_launch<S, float, 0>(ctx, d_gtab, L, M, Upad, lay, d_in, n_in, d_out, n_out, stream);
    }
}

}  // namespace

// G[k0][q][u] = bank_k0[M*u + q - s_k0],  bank_k0[t] = taps[L*(T-1-t) + (k0*M mod L)],  s_k0 = floor(k0*M/L) + lead;
// tf floats per tap, [L][M][slide_upad(M, T)] taps in all.
std::vector<float> slide_table(const float *taps, size_t tf, size_t L, size_t M, size_t T, size_t lead) {
    const size_t Upad = (size_t)slide_upad(M, T);
    std::vector<float> g(L * M * Upad * tf, 0.0f);
    for (size_t k0 = 0; k0 < L; k0++) {
        const size_t bank = (k0 * M) % L, s = (k0 * M) / L + lead;
        for (size_t q = 0; q < M; q++)
            for (size_t u = 0; u < Upad; u++) {
                const long long t = (long long)(M * u + q) - (long long)s;
                if (t < 0 || t >= (long long)T) continue;
                for (size_t c = 0; c < tf; c++)
                    g[((k0 * M + q) * Upad + u) * tf + c] = taps[(L * (T - 1 - (size_t)t) + bank) * tf + c];
            }
    }
    return g;
}

// The phase table of the FIR (L = 1, M = D, shift D-1) followed by the plain reversed taps g[t] = taps[N-1-t]
// (read by fir_naive_kernel and the tensor-core kernel).
int32_t fir_direct_prepare(b2s_fir *f) {
    b2s_ctx *ctx = f->ctx;
    const size_t N = f->ntaps, D = f->decim, tf = kind_tap_floats(f->kind);
    f->Upad = slide_upad(D, N);
    std::vector<float> h = slide_table(f->taps_host.data(), tf, 1, D, N, D - 1);
    for (size_t t = 0; t < N; t++)
        for (size_t c = 0; c < tf; c++) h.push_back(f->taps_host[(N - 1 - t) * tf + c]);
    B2S_TRY(f->d_ptaps.upload(ctx, h.data(), h.size(), "FIR taps"));
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

bool resamp_slide_supported(size_t L, size_t M, size_t T, size_t item_bytes) {
    const size_t Upad = (size_t)slide_upad(M, T);
    // worthwhile only while the zero padding of the per-phase taps stays small (T/M taps per phase row)
    if (Upad * M > 2 * (T + M) + 16) return false;
    size_t smem = slide_layout(L, M, Upad, item_bytes, sizeof(float)).smem;
    // L = 1 stages its outputs in the phase rows, yet the budget counts a staging of THREADS*(R+1) items for it as for
    // L >= 5: which plans take this kernel instead of resamp_kernel, whose summation order differs, decides their
    // output bits, and this keeps that set fixed.
    if (L == 1) smem += round_up(kThreads * (kR + 1) * item_bytes, 16);
    return smem <= kRsSmemMax;
}

int32_t resamp_slide_launch(b2s_ctx *ctx, b2s_kind kind, const float *d_gtab, size_t L, size_t M, size_t T,
                            const void *d_in, size_t n_in, void *d_out, size_t n_out, cudaStream_t stream) {
    const int Upad = slide_upad(M, T);
    if (kind == B2S_F32_F32)
        return resamp_launch_typed<float>(ctx, d_gtab, (int)L, (int)M, Upad, d_in, n_in, d_out, n_out, stream);
    return resamp_launch_typed<float2>(ctx, d_gtab, (int)L, (int)M, Upad, d_in, n_in, d_out, n_out, stream);
}
