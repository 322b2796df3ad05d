// iir.cu -- futuredsp::IirFilter (crates/futuredsp/src/iir.rs:33-178), the core of blocks::Iir (src/blocks/iir.rs).
//
// The reference's recurrence (iir.rs:136-164), per output k of a call:
//     o = 0;  o += b[j] * i[k + n_b - 1 - j]  (j = 0..n_b);  o += a[j] * memory[j]  (j = 0..n_a)
//     memory shifts by one, memory[0] = o
// with `memory` first filled with the stream's first n_a INPUT samples (memory[j] = x[j], not consumed, :102-129).
//
// Two kernels:
//   iir_seq_kernel   one thread walks the recurrence with un-fused IEEE mul/add in the reference's order: bit-identical
//                    to the reference for f32 and f64 (denormals and non-finite values included).  The other threads
//                    of the CTA stage input and output tiles through shared memory.
//   iir_scan_kernel  (f32, stable filters, 1 <= n_a <= 8, n_b <= 64) a single-pass chained scan.  The state after
//                    output k is s_k = A s_{k-1} + e_0 u_k (A: companion matrix of a, u_k: the b-sum), so a segment of
//                    L outputs maps a start state S to A^L S + E, E being the segment's zero-start end state.  A CTA
//                    takes a tile of T = 256 x 16 outputs: each thread runs its 16 outputs from zero state, a
//                    Kogge-Stone scan over threads composes the E's, decoupled look-back over earlier tiles gives the
//                    tile's true start state, and each thread then re-runs its 16 outputs from its true start state
//                    with the reference's operations.  Every power of A is computed in f64 at plan time.
#include <cmath>
#include <vector>

#include "fir.cuh"

namespace {

// ---- sequential kernel -------------------------------------------------------------------------------------------
constexpr int kSeqThreads = 256, kSeqTile = 2048;
constexpr size_t kSeqMaxTaps = 2048;               // n_a and n_b each (shared-memory staging)

template <typename T> __device__ __forceinline__ T mul_rn(T a, T b);
template <typename T> __device__ __forceinline__ T add_rn(T a, T b);
template <> __device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
template <> __device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
template <> __device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
template <> __device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

// memory is kept as a ring: memory[j] = ring[(h + j) mod n_a]; the shift of :155-160 is h -= 1, ring[h] = o.
template <typename T>
__global__ void __launch_bounds__(kSeqThreads)
iir_seq_kernel(const T *__restrict__ in, T *__restrict__ out, long long n, const T *__restrict__ a_taps, int n_a,
               const T *__restrict__ b_taps, int n_b, T *mem) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T *sb = reinterpret_cast<T *>(smem_raw), *sa = sb + n_b, *ring = sa + n_a, *xs = ring + n_a;
    T *ys = xs + kSeqTile + n_b - 1;
    for (int j = threadIdx.x; j < n_b; j += blockDim.x) sb[j] = b_taps[j];
    for (int j = threadIdx.x; j < n_a; j += blockDim.x) { sa[j] = a_taps[j]; ring[j] = mem[j]; }
    int h = 0;
    for (long long k0 = 0; k0 < n; k0 += kSeqTile) {
        const int nk = (int)min((long long)kSeqTile, n - k0);
        __syncthreads();                                  // previous tile's ys stored, xs free
        for (int i = threadIdx.x; i < nk + n_b - 1; i += blockDim.x) xs[i] = in[k0 + i];
        __syncthreads();
        // the b-sums (:142-145) do not depend on the recurrence: every thread forms some, same operations and order
        for (int k = threadIdx.x; k < nk; k += blockDim.x) {
            T o = T(0);
            for (int j = 0; j < n_b; j++) o = add_rn(o, mul_rn(sb[j], xs[k + n_b - 1 - j]));
            ys[k] = o;
        }
        __syncthreads();
        if (threadIdx.x == 0 && n_a) {
            for (int k = 0; k < nk; k++) {
                T o = ys[k];
                int idx = h;
                for (int j = 0; j < n_a; j++) {
                    o = add_rn(o, mul_rn(sa[j], ring[idx]));
                    idx = idx + 1 == n_a ? 0 : idx + 1;
                }
                h = h == 0 ? n_a - 1 : h - 1;
                ring[h] = o;
                ys[k] = o;
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < nk; i += blockDim.x) out[k0 + i] = ys[i];
    }
    if (threadIdx.x == 0)
        for (int j = 0; j < n_a; j++) mem[j] = ring[(h + j) % n_a];
}

// ---- chained-scan kernel (f32) ----------------------------------------------------------------------------------
constexpr int kScanThreads = 256, kScanR = 16, kScanTile = kScanThreads * kScanR;
constexpr int kScanMaxA = 8, kScanMaxB = 64;
constexpr int kLookMax = 1024;                     // look-back depth with tabulated A^(T m); deeper waits for a prefix
constexpr unsigned kAgg = 1, kPre = 2;             // status word: (seq << 2) | kind
constexpr unsigned long long kSpinTimeoutNs = 4000000000ull;

// power tables, row-major NA x NA each: thr[t] = A^(R t) for t = 0..kScanThreads, tile[m] = A^(T m) for m = 0..kLookMax
struct ScanTables { const float *thr; const float *tile; };

__device__ __forceinline__ unsigned ld_acquire(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(unsigned *p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

template <int NA>
__device__ __forceinline__ void matvec_acc(float (&acc)[NA], const float *__restrict__ M, const float (&v)[NA]) {
#pragma unroll
    for (int i = 0; i < NA; i++) {
        float s = acc[i];
#pragma unroll
        for (int c = 0; c < NA; c++) s = fmaf(__ldg(M + i * NA + c), v[c], s);
        acc[i] = s;
    }
}

template <int NA>
__global__ void __launch_bounds__(kScanThreads, 3)
iir_scan_kernel(const float *__restrict__ in, float *__restrict__ out, long long n, const float *__restrict__ a_taps,
                const float *__restrict__ b_taps, int n_b, float *mem, ScanTables tab, unsigned long long *counter,
                unsigned long long tile_base, unsigned *status, float *agg, float *pre, unsigned seq,
                unsigned *err) {
    __shared__ float xs[kScanTile + kScanMaxB];
    __shared__ float us[kScanTile + kScanTile / kScanR];   // padded: element k at k + k / 16
    __shared__ float st[kScanThreads][NA];
    __shared__ float sb[kScanMaxB], sa[NA], s_in[NA];
    __shared__ long long s_tile;
    const int t = threadIdx.x;
    if (t == 0) s_tile = (long long)(atomicAdd(counter, 1ull) - tile_base);   // tiles start in launch order
    if (t < n_b) sb[t] = b_taps[t];
    if (t < NA) sa[t] = a_taps[t];
    __syncthreads();
    const long long tile = s_tile, k0 = tile * kScanTile;
    const int nk = (int)min((long long)kScanTile, n - k0);
    const long long n_in_tile = nk + n_b - 1;
    for (int i = t; i < n_in_tile; i += kScanThreads) xs[i] = in[k0 + i];
    __syncthreads();
    // b-sums in the reference's order (:139-145), coalesced over k = t + 256 r
#pragma unroll 4
    for (int r = 0; r < kScanR; r++) {
        const int k = t + r * kScanThreads;
        float o = 0.0f;
        for (int j = 0; j < n_b; j++) o = __fadd_rn(o, __fmul_rn(sb[j], xs[k + n_b - 1 - j]));
        us[k + (k >> 4)] = o;
    }
    __syncthreads();
    // each thread: its 16 consecutive outputs from zero state -> zero-start end state E
    float u[kScanR], a[NA], m[NA];
#pragma unroll
    for (int j = 0; j < NA; j++) { a[j] = sa[j]; m[j] = 0.0f; }
#pragma unroll
    for (int r = 0; r < kScanR; r++) {
        u[r] = us[t * (kScanR + 1) + r];
        float y = u[r];
#pragma unroll
        for (int j = 0; j < NA; j++) y = fmaf(a[j], m[j], y);
#pragma unroll
        for (int j = NA - 1; j > 0; j--) m[j] = m[j - 1];
        m[0] = y;
    }
    // Kogge-Stone over threads: F_t <- F_t + A^(R d) F_{t-d}
#pragma unroll 1
    for (int d = 1; d < kScanThreads; d <<= 1) {
#pragma unroll
        for (int j = 0; j < NA; j++) st[t][j] = m[j];
        __syncthreads();
        if (t >= d) {
            float v[NA];
#pragma unroll
            for (int j = 0; j < NA; j++) v[j] = st[t - d][j];
            matvec_acc<NA>(m, tab.thr + (size_t)d * NA * NA, v);
        }
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < NA; j++) st[t][j] = m[j];
    __syncthreads();
    // tile start state: decoupled look-back (warp 0)
    if (t < 32) {
        const int lane = t;
        float tot[NA];
        if (tile == 0) {
#pragma unroll
            for (int j = 0; j < NA; j++) tot[j] = lane == 0 ? mem[j] : 0.0f;
        } else {
            if (lane == 0) {                                  // publish the aggregate first
#pragma unroll
                for (int j = 0; j < NA; j++) __stcg(agg + tile * NA + j, st[kScanThreads - 1][j]);
                __threadfence();
                st_release(status + tile, (seq << 2) | kAgg);
            }
            float acc[NA];
#pragma unroll
            for (int j = 0; j < NA; j++) acc[j] = 0.0f;
            const unsigned long long t0 = globaltimer();
            bool timed_out = false;
            for (int base = 0;;) {
                const int mm = base + lane;                   // this lane looks at tile - 1 - mm
                const long long pred = tile - 1 - mm;
                const bool valid = pred >= 0 && mm < kLookMax;
                const bool must_pre = mm == kLookMax - 1;     // at the table's end only a prefix will do
                unsigned kind = 0;
                if (valid) {
                    for (;;) {
                        const unsigned s = ld_acquire(status + pred);
                        if ((s >> 2) == (seq & 0x3FFFFFFFu)) kind = s & 3u;
                        if (kind == kPre || (kind == kAgg && !must_pre)) break;
                        if (timed_out || globaltimer() - t0 > kSpinTimeoutNs) { timed_out = true; kind = kPre; break; }
                        __nanosleep(64);
                    }
                }
                const unsigned pre_mask = __ballot_sync(0xffffffffu, valid && kind == kPre);
                const int first = pre_mask ? __ffs(pre_mask) - 1 : 32;
                if (valid && lane <= first) {
                    float v[NA];
                    const float *src = (lane == first ? pre : agg) + pred * NA;
#pragma unroll
                    for (int j = 0; j < NA; j++) v[j] = __ldcg(src + j);
                    matvec_acc<NA>(acc, tab.tile + (size_t)mm * NA * NA, v);     // S_in = sum_m A^(T m) x_{tile-1-m}
                }
                if (pre_mask) break;
                base += 32;
            }
            if (__any_sync(0xffffffffu, timed_out) && lane == 0) atomicOr(err, 2u);
#pragma unroll
            for (int j = 0; j < NA; j++) {
                float s = acc[j];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                tot[j] = s;
            }
        }
        if (lane == 0) {                                      // inclusive prefix of this tile: F_255 + A^T S_in
            float p[NA];
#pragma unroll
            for (int j = 0; j < NA; j++) { p[j] = st[kScanThreads - 1][j]; s_in[j] = tot[j]; }
            matvec_acc<NA>(p, tab.thr + (size_t)kScanThreads * NA * NA, tot);
#pragma unroll
            for (int j = 0; j < NA; j++) __stcg(pre + tile * NA + j, p[j]);
            __threadfence();
            st_release(status + tile, (seq << 2) | kPre);
        }
    }
    __syncthreads();
    // this thread's true start state: F_{t-1} + A^(R t) S_in, then the reference's recurrence (:148-160)
    float sin_[NA];
#pragma unroll
    for (int j = 0; j < NA; j++) { sin_[j] = s_in[j]; m[j] = t > 0 ? st[t - 1][j] : 0.0f; }
    matvec_acc<NA>(m, tab.thr + (size_t)t * NA * NA, sin_);
#pragma unroll
    for (int r = 0; r < kScanR; r++) {
        float y = u[r];
#pragma unroll
        for (int j = 0; j < NA; j++) y = __fadd_rn(y, __fmul_rn(a[j], m[j]));
#pragma unroll
        for (int j = NA - 1; j > 0; j--) m[j] = m[j - 1];
        m[0] = y;
        us[t * (kScanR + 1) + r] = y;
    }
    __syncthreads();
    for (int k = t; k < nk; k += kScanThreads) out[k0 + k] = us[k + (k >> 4)];
    if (k0 + nk == n && t < NA) {                             // the tile holding output n-1 leaves the new memory
        const long long idx = n - 1 - t;
        mem[t] = idx >= k0 ? us[(idx - k0) + ((idx - k0) >> 4)] : s_in[t - nk];
    }
}

// f64 companion-matrix helpers (plan time)
using Mat = std::vector<double>;
Mat mat_mul(const Mat &x, const Mat &y, int d) {
    Mat z((size_t)d * d, 0.0);
    for (int i = 0; i < d; i++)
        for (int k = 0; k < d; k++)
            for (int j = 0; j < d; j++) z[i * d + j] += x[i * d + k] * y[k * d + j];
    return z;
}
Mat companion(const std::vector<double> &a) {
    const int d = (int)a.size();
    Mat m((size_t)d * d, 0.0);
    for (int j = 0; j < d; j++) m[j] = a[j];
    for (int i = 1; i < d; i++) m[i * d + i - 1] = 1.0;
    return m;
}
double mat_norm_inf(const Mat &x, int d) {
    double best = 0;
    for (int i = 0; i < d; i++) {
        double s = 0;
        for (int j = 0; j < d; j++) s += std::fabs(x[i * d + j]);
        best = std::max(best, s);
    }
    return best;
}

}  // namespace

struct b2s_iir {
    b2s_ctx *ctx = nullptr;
    bool f64 = false;
    size_t n_a = 0, n_b = 0;
    std::vector<double> a, b;                  // taps as given (f32 plans hold f32 values)
    b2s_algo algo_req = B2S_ALGO_AUTO, algo = B2S_ALGO_DIRECT;
    bool scan_ok = false;                      // plan admitted to the chained scan
    size_t fill = 0;                           // memory items filled so far (data-independent host mirror)
    Buf<char> d_a, d_b, d_mem;                 // T = float or double (f64) taps and filter memory
    PlanPtr<b2s_fir> fir;                      // AUTO with n_a == 0: the FIR plan with taps = b
    // scan state
    Buf<float> d_tables;
    Buf<unsigned long long> d_counter;
    unsigned long long tiles_launched = 0;
    unsigned seq = 0;
    Buf<unsigned> d_status;
    Buf<float> d_agg, d_pre;
    size_t status_tiles = 0;
};

namespace {

// 1 <= n_a <= 8, n_b <= 64 and max|pole| < 1 - 6.6e-6, decided in f64 as ||A^(2^20)|| < 1e-3
bool scan_admits(const b2s_iir *f) {
    if (f->f64 || f->n_a < 1 || f->n_a > (size_t)kScanMaxA || f->n_b > (size_t)kScanMaxB) return false;
    const int d = (int)f->n_a;
    Mat p = companion(f->a);
    for (int i = 0; i < 20; i++) {
        p = mat_mul(p, p, d);
        const double nrm = mat_norm_inf(p, d);
        if (!std::isfinite(nrm)) return false;
        if (nrm > 1e30) return false;
    }
    return mat_norm_inf(p, d) < 1e-3;
}

int32_t scan_prepare(b2s_iir *f) {
    if (f->d_tables) return B2S_OK;
    b2s_ctx *ctx = f->ctx;
    const int d = (int)f->n_a, dd = d * d;
    const size_t n_thr = kScanThreads + 1, n_tile = kLookMax + 1;
    std::vector<float> h((n_thr + n_tile) * dd);
    Mat eye((size_t)dd, 0.0);
    for (int i = 0; i < d; i++) eye[i * d + i] = 1.0;
    const Mat A = companion(f->a);
    Mat AR = eye;
    for (int i = 0; i < kScanR; i++) AR = mat_mul(AR, A, d);
    Mat p = eye;
    for (size_t t = 0; t < n_thr; t++) {                     // A^(R t)
        for (int i = 0; i < dd; i++) h[t * dd + i] = (float)p[i];
        p = mat_mul(p, AR, d);
    }
    Mat AT = eye;
    for (int i = 0; i < kScanThreads; i++) AT = mat_mul(AT, AR, d);
    p = eye;
    for (size_t m = 0; m < n_tile; m++) {                    // A^(T m)
        for (int i = 0; i < dd; i++) h[(n_thr + m) * dd + i] = (float)p[i];
        p = mat_mul(p, AT, d);
    }
    Buf<float> tables;
    Buf<unsigned long long> counter;
    B2S_TRY(tables.upload(ctx, h.data(), h.size(), "iir scan tables"));   // pageable h is staged before the call returns
    B2S_TRY(counter.alloc(ctx, 1, "iir scan counter"));
    B2S_CUDA(ctx, cudaMemsetAsync(counter.get(), 0, sizeof(unsigned long long), ctx->stream));
    f->d_tables = std::move(tables);                         // the plan is scan-ready only with both
    f->d_counter = std::move(counter);
    f->tiles_launched = 0;
    return B2S_OK;
}

int32_t scan_reserve(b2s_iir *f, size_t tiles) {
    if (tiles <= f->status_tiles) return B2S_OK;
    b2s_ctx *ctx = f->ctx;
    f->status_tiles = 0;
    const size_t cap = std::max<size_t>(tiles, 64);
    B2S_TRY(f->d_status.reserve(ctx, cap, "iir scan status"));
    B2S_TRY(f->d_agg.reserve(ctx, cap * f->n_a, "iir scan aggregates"));
    B2S_TRY(f->d_pre.reserve(ctx, cap * f->n_a, "iir scan prefixes"));
    // tag 0 never matches a call's sequence
    B2S_CUDA(ctx, cudaMemsetAsync(f->d_status.get(), 0, cap * sizeof(unsigned), ctx->stream));
    f->status_tiles = cap;
    return B2S_OK;
}

template <int NA>
void scan_launch_na(b2s_iir *f, const float *in, float *out, long long n, unsigned grid, cudaStream_t st) {
    ScanTables tab{f->d_tables.get(), f->d_tables.get() + (size_t)(kScanThreads + 1) * NA * NA};
    iir_scan_kernel<NA><<<grid, kScanThreads, 0, st>>>(in, out, n, (const float *)f->d_a.get(), (const float *)f->d_b.get(),
                                                       (int)f->n_b, (float *)f->d_mem.get(), tab, f->d_counter.get(),
                                                       f->tiles_launched, f->d_status.get(), f->d_agg.get(), f->d_pre.get(), f->seq,
                                                       f->ctx->d_status);
}

int32_t scan_launch(b2s_iir *f, const void *d_in, void *d_out, size_t n) {
    b2s_ctx *ctx = f->ctx;
    const size_t tiles = ceil_div(n, (size_t)kScanTile);
    int32_t rc = scan_prepare(f);
    if (rc != B2S_OK) return rc;
    if ((rc = scan_reserve(f, tiles)) != B2S_OK) return rc;
    f->seq = (f->seq + 1) & 0x3FFFFFFFu;
    if (f->seq == 0) f->seq = 1;
    const float *in = (const float *)d_in;
    float *out = (float *)d_out;
    const unsigned grid = (unsigned)tiles;
    cudaStream_t st = ctx->stream;
    switch (f->n_a) {
        case 1: scan_launch_na<1>(f, in, out, (long long)n, grid, st); break;
        case 2: scan_launch_na<2>(f, in, out, (long long)n, grid, st); break;
        case 3: scan_launch_na<3>(f, in, out, (long long)n, grid, st); break;
        case 4: scan_launch_na<4>(f, in, out, (long long)n, grid, st); break;
        case 5: scan_launch_na<5>(f, in, out, (long long)n, grid, st); break;
        case 6: scan_launch_na<6>(f, in, out, (long long)n, grid, st); break;
        case 7: scan_launch_na<7>(f, in, out, (long long)n, grid, st); break;
        default: scan_launch_na<8>(f, in, out, (long long)n, grid, st); break;
    }
    f->tiles_launched += tiles;
    ctx->flag_ops++;                                         // b2s_ctx_sync reports a look-back time-out
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

template <typename T>
int32_t seq_launch(b2s_iir *f, const void *d_in, void *d_out, size_t n) {
    constexpr size_t max_smem = (kSeqMaxTaps + 2 * kSeqMaxTaps + kSeqTile + kSeqMaxTaps - 1 + kSeqTile) * sizeof(T);
    B2S_TRY(smem_optin<iir_seq_kernel<T>>(f->ctx, max_smem));
    const size_t smem = (f->n_b + 2 * f->n_a + kSeqTile + f->n_b - 1 + kSeqTile) * sizeof(T);
    iir_seq_kernel<T><<<1, kSeqThreads, smem, f->ctx->stream>>>((const T *)d_in, (T *)d_out, (long long)n,
                                                               (const T *)f->d_a.get(), (int)f->n_a, (const T *)f->d_b.get(),
                                                               (int)f->n_b, (T *)f->d_mem.get());
    B2S_CHECK_LAUNCH(f->ctx);
    return B2S_OK;
}

void resolve_algo(b2s_iir *f) {
    if (f->algo_req == B2S_ALGO_SCAN) f->algo = B2S_ALGO_SCAN;           // set_algo checked admission
    else if (f->algo_req == B2S_ALGO_AUTO && f->scan_ok) f->algo = B2S_ALGO_SCAN;
    else if (f->algo_req == B2S_ALGO_AUTO && f->fir) f->algo = (b2s_algo)b2s_fir_get_algo(f->fir.get());
    else f->algo = B2S_ALGO_DIRECT;
}

template <typename T>
int32_t iir_plan(b2s_ctx *ctx, const T *a_taps, size_t n_a, const T *b_taps, size_t n_b, bool f64, b2s_iir **out) {
    if (!ctx || !out || (n_a && !a_taps) || !b_taps) return b2s_fail(ctx, B2S_EINVAL, "b2s_iir_plan: NULL argument");
    *out = nullptr;
    if (n_b == 0) return b2s_fail(ctx, B2S_EINVAL, "b2s_iir_plan: n_b must be > 0 (iir.rs:132)");
    if (n_a > kSeqMaxTaps || n_b > kSeqMaxTaps)
        return b2s_fail(ctx, B2S_EUNSUPPORTED, "b2s_iir_plan: at most %zu a taps and %zu b taps", kSeqMaxTaps, kSeqMaxTaps);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_iir> f(new b2s_iir());
    f->ctx = ctx; f->f64 = f64; f->n_a = n_a; f->n_b = n_b;
    f->a.assign(a_taps, a_taps + n_a);
    f->b.assign(b_taps, b_taps + n_b);
    const size_t sz = sizeof(T);
    B2S_TRY(f->d_a.alloc(ctx, std::max<size_t>(n_a, 1) * sz, "iir a taps"));
    B2S_TRY(f->d_b.upload(ctx, (const char *)b_taps, n_b * sz, "iir b taps"));
    B2S_TRY(f->d_mem.alloc(ctx, std::max<size_t>(n_a, 1) * sz, "iir memory"));
    if (n_a) B2S_CUDA(ctx, cudaMemcpyAsync(f->d_a.get(), a_taps, n_a * sz, cudaMemcpyHostToDevice, ctx->stream));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    f->scan_ok = scan_admits(f.get());
    if (n_a == 0) {
        b2s_fir *fir = nullptr;
        B2S_TRY(f64 ? b2s_fir_plan_f64_f64(ctx, (const double *)(const void *)b_taps, n_b, 1, &fir)
                    : b2s_fir_plan_f32_f32(ctx, (const float *)(const void *)b_taps, n_b, 1, &fir));
        f->fir.reset(fir);
    }
    resolve_algo(f.get());
    *out = f.release();
    return B2S_OK;
}

// (consumed, produced, status) of taps_accessor_work (iir.rs:90-177); advances the fill count and reports how many
// memory items this call fills (from d_in[fill_from ..)).
void iir_counts(b2s_iir *f, size_t n_in, size_t n_out_cap, size_t *consumed, size_t *produced, int32_t *status,
                size_t *fill_from, size_t *fill_n) {
    const int32_t st_empty = n_out_cap == 0 ? B2S_BOTH_SUFFICIENT : B2S_INSUFFICIENT_INPUT;
    *consumed = *produced = 0; *status = st_empty; *fill_from = f->fill; *fill_n = 0;
    if (n_in == 0) return;                                                   // :90-100
    if (f->fill < f->n_a) {                                                  // :102-118
        const size_t to = std::max(f->fill, std::min(f->n_a, n_in));
        *fill_n = to - f->fill;
        f->fill = to;
        if (f->fill < f->n_a) return;
    }
    if (*fill_n == n_in) return;                                             // :119-129
    const size_t n = std::min(sat_sub(n_in + 1, f->n_b), n_out_cap);        // :136
    *consumed = *produced = n;
    if (n == n_in && n == n_out_cap) *status = B2S_BOTH_SUFFICIENT;         // :166-177
    else if (n < n_in) *status = B2S_INSUFFICIENT_OUTPUT;
    else *status = B2S_INSUFFICIENT_INPUT;
}

}  // namespace

extern "C" {

int32_t b2s_iir_plan_f32(b2s_ctx *ctx, const float *a_taps, size_t n_a, const float *b_taps, size_t n_b, b2s_iir **out) {
    return iir_plan<float>(ctx, a_taps, n_a, b_taps, n_b, false, out);
}
int32_t b2s_iir_plan_f64(b2s_ctx *ctx, const double *a_taps, size_t n_a, const double *b_taps, size_t n_b, b2s_iir **out) {
    return iir_plan<double>(ctx, a_taps, n_a, b_taps, n_b, true, out);
}

void b2s_iir_destroy(b2s_iir *f) { PlanDeleter<b2s_iir>()(f); }

size_t b2s_iir_length(const b2s_iir *f) { return f ? f->n_b : 0; }

int32_t b2s_iir_set_algo(b2s_iir *f, b2s_algo algo) {
    if (!f) return b2s_fail(nullptr, B2S_EINVAL, "iir is NULL");
    if (algo != B2S_ALGO_AUTO && algo != B2S_ALGO_DIRECT && algo != B2S_ALGO_SCAN)
        return b2s_fail(f->ctx, B2S_EUNSUPPORTED, "IIR filters have the AUTO, DIRECT and SCAN algorithms (got %d)", (int)algo);
    if (algo == B2S_ALGO_SCAN && !f->scan_ok)
        return b2s_fail(f->ctx, B2S_EUNSUPPORTED,
                        "SCAN needs f32, 1..8 a taps, at most 64 b taps and a stable filter (max|pole| < 1 - 6.6e-6); "
                        "plan has %s, n_a %zu, n_b %zu", f->f64 ? "f64" : "f32", f->n_a, f->n_b);
    f->algo_req = algo;
    resolve_algo(f);
    return B2S_OK;
}
int32_t b2s_iir_get_algo(const b2s_iir *f) { return f ? (int32_t)f->algo : B2S_EINVAL; }

int32_t b2s_iir_exec(b2s_iir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap, size_t *consumed,
                     size_t *produced, int32_t *status) {
    if (!f || !consumed || !produced || !status)
        return b2s_fail(f ? f->ctx : nullptr, B2S_EINVAL, "b2s_iir_exec: NULL argument");
    if (n_in && !d_in) return b2s_fail(f->ctx, B2S_EINVAL, "b2s_iir_exec: NULL input");
    const size_t isz = f->f64 ? 8 : 4;
    const size_t fill_before = f->fill;
    size_t fill_from, fill_n;
    iir_counts(f, n_in, n_out_cap, consumed, produced, status, &fill_from, &fill_n);
    const size_t n = *produced;
    if (n && !d_out) { f->fill = fill_before; *consumed = *produced = 0; return b2s_fail(f->ctx, B2S_EINVAL, "b2s_iir_exec: NULL output"); }
    if (n) {
        const char *ib = (const char *)d_in, *ob = (const char *)d_out;
        if (ob < ib + n_in * isz && ib < ob + n * isz) {
            f->fill = fill_before; *consumed = *produced = 0;
            return b2s_fail(f->ctx, B2S_EINVAL, "b2s_iir_exec: input and output slices overlap");
        }
    }
    DeviceGuard g(f->ctx->device);
    NvtxRange nvtx("b2s_iir_exec");
    cudaStream_t st = f->ctx->stream;
    if (fill_n)                                                              // memory[j] = x[j] (:116)
        B2S_CUDA(f->ctx, cudaMemcpyAsync(f->d_mem.get() + fill_from * isz, (const char *)d_in + fill_from * isz,
                                         fill_n * isz, cudaMemcpyDeviceToDevice, st));
    if (n == 0) return B2S_OK;
    if (f->fir && f->algo_req == B2S_ALGO_AUTO) {                            // n_a == 0: the same sum on the FIR plan
        size_t c = 0, p = 0; int32_t s = 0;
        return b2s_fir_exec(f->fir.get(), d_in, n_in, d_out, n, &c, &p, &s);
    }
    if (f->algo == B2S_ALGO_SCAN) return scan_launch(f, d_in, d_out, n);
    return f->f64 ? seq_launch<double>(f, d_in, d_out, n) : seq_launch<float>(f, d_in, d_out, n);
}

}  // extern "C"
