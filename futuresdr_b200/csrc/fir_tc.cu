// fir_tc.cu -- wgmma (Hopper tensor core) FIR for 16..257 real taps on sm_90a.
//
// Computes the same  o[k] = sum_t i[k+t] * taps[N-1-t]  as crates/futuredsp/src/fir.rs:77-88
// (Complex<f32> or f32 samples, f32 taps; decimating_fir.rs:80-92 for a decimation D | 128: the epilogue keeps
// the output phases D-1 mod D) as a block-Toeplitz GEMM:
//
//      D[p][c] = sum_kappa A[p][kappa] * B[c][kappa]            (M = 128, N = 128, K = 128*DK <= 384)
//      A[p][kappa] = g[kappa - p]   (g[t] = taps[N-1-t], zero outside [0,N))   -- "taps, Toeplitz"
//      B[c][kappa] = w_c[kappa]     (column c = one 128-sample block of the re- or im-stream,
//                                    extended by the following blocks)         -- "samples"
//      => D[p][c] = y[128*block(c) + p]
//
//  * A is constant and Toeplitz, so it is stored ALIASED: the rows are kept in reversed order
//    (row p' = 127 - p), which makes A[p'][kappa] a function of kappa + p' alone.  In the
//    no-swizzle K-major layout (8x8 core matrices of 128 bytes) core matrix (row group a, K group j)
//    then only depends on a + j, and one descriptor with LBO = SBO = 128 bytes walks a strip of
//    K/8 + 15 core matrices (~8 KiB per precision instead of 96 KiB for the full 128 x 384 matrix).
//  * FP32 accuracy on bf16 tensor cores: x = x_hi + x_lo, g = g_hi + g_lo (bf16 each) and
//    x*g ~= x_hi*g_hi + x_lo*g_hi + x_hi*g_lo, three bf16 wgmma accumulating in FP32 registers.
//    Dropped terms are O(2^-17) relative per product (DESIGN.md "tensor FIR numerics").
//  * B rows are K-major, 128-byte swizzled.  K-block d of row (stream, block b) is row
//    (stream, block b+d): a shifted view of the same tile.  Rows are stored so that the shift
//    is a whole 8-row swizzle atom: physical atom gamma holds blocks {gamma + 16*jb}; the view
//    for shift d starts at atom d (descriptor base + 1024*d bytes).  Atoms 16, 17 duplicate the
//    rows they alias (12 % extra conversion work, no extra HBM traffic).
//  * 5 warpgroups, one persistent CTA per SM, everything handed over with mbarriers; setmaxnreg moves registers
//    from the converters and the loader to the math warpgroups:
//      warp 16    TMA loader : cp.async.bulk of the raw f32 samples into a 6 x 8 KiB ring (warps 17-19 only
//                              complete the loader warpgroup and exit)
//      warps 8-15 converters : LDS.128 -> bf16 hi/lo split (cvt.rn.bf16x2) -> swizzled st.shared
//                              into one of two 72 KiB operand stages
//      warps 0-7  two math warpgroups, 64 output phases (M rows) each: 3 wgmma.m64n128k16 per K-step, only over
//                 the K-steps whose Toeplitz slice holds a tap for the warpgroup's phases (20 of 24 at 256 taps),
//                 into 64 FP32 accumulator registers per thread, stored straight from the registers.  The two
//                 g_hi products take their A operand from registers (fragments loaded once per kernel), g_lo * x_hi
//                 from the strip in shared memory.
#include <cuda_bf16.h>

#include <algorithm>
#include <climits>
#include <cstdlib>
#include <type_traits>

#include "fir.cuh"

namespace {

constexpr int kStages = 2;                  // bf16 operand stages (72 KiB each)
#ifndef B2S_RAW_SLOTS
#define B2S_RAW_SLOTS 6
#endif
constexpr int kRawSlots = B2S_RAW_SLOTS;    // raw f32 staging ring, 8 KiB per slot (TMA bulk copies)
constexpr int kRawSlotBytes = 8192;
constexpr int kNumProducerThreads = 256;    // 8 converter warps
constexpr int kNumMathThreads = 256;        // 2 warpgroups: wgmma + epilogue
constexpr int kNumLoaderThreads = 128;      // loader warpgroup: one TMA warp, three that exit (setmaxnreg is per warpgroup)
constexpr int kThreadsTC = kNumMathThreads + kNumProducerThreads + kNumLoaderThreads;   // 640
constexpr int kProdWarps = kNumProducerThreads / 32;
constexpr int kMathWarps = kNumMathThreads / 32;
constexpr int kProdWarp0 = kMathWarps;               // warps 8..15 converters
constexpr int kTmaWarp = kProdWarp0 + kProdWarps;    // warp 16
// Registers per thread: __launch_bounds__(640, 1) gives every thread 96 (65536 / 640, in units of 8).  The math
// warpgroups hold 64 accumulators, 80 registers of g_hi fragments (4 per K-step) and the epilogue's addresses, so they
// take what the converters (48 suffice) and the loader give back; the CTA's allocation must cover
// the sum or setmaxnreg.inc never returns.  kRegsAtLaunch assumes ptxas gives the kernel exactly that count at entry
// (-Xptxas -v: "Used 96 registers"); a lower entry count would shrink the pool below the budget, so fir_tc_prepare
// refuses the plan if the built kernel reports any other count.
constexpr int kRegsAtLaunch = 65536 / kThreadsTC / 8 * 8;
constexpr int kMathRegs = 176, kProdRegs = 48, kLoaderRegs = 24;
static_assert(kNumMathThreads * kMathRegs + kNumProducerThreads * kProdRegs + kNumLoaderThreads * kLoaderRegs <=
              kThreadsTC * kRegsAtLaunch, "setmaxnreg budget exceeds the CTA's register allocation");
constexpr int kSchedSlots = 64;              // tile counters per plan (launches of a plan that may be in flight at once)
constexpr int kAtomsOut = 16;                // N = 128 columns = 16 swizzle atoms of 8 rows
constexpr int kMaxDK = 3;                    // K <= 384
// K-steps one math warpgroup issues per tile: its 64 phases start on a multiple of 16 and lead + ntaps <= 128*DK - 127,
// so its tap columns span at most floor((63 + 128*kMaxDK - 128) / 16) + 1 = 20 slices of 16
constexpr int kMaxKSteps = (63 + 128 * kMaxDK - 128) / 16 + 1;
constexpr int kSplitBytesMax = (kAtomsOut + kMaxDK - 1) * 1024 * 2;   // per split: 2 K-chunks x 18 atoms
constexpr int kStageBytes = 2 * kSplitBytesMax;                       // hi + lo = 72 KiB
constexpr int kACores = kMaxDK * 16 + 15;    // core matrices of the aliased Toeplitz strip (K/8 + 128/8 - 1)
constexpr int kABytes = kACores * 128;       // per precision (hi, lo)
constexpr int kSmemTC = kStages * kStageBytes + kRawSlots * kRawSlotBytes + 2 * kABytes + 1024 /*align*/ + 256 /*barriers*/;
static_assert(8 * (2 * kStages + 2 * kRawSlots) + 16 + 4 * kStages <= 256, "barriers and tile numbers exceed their 256 bytes");
static_assert(kSmemTC <= 227 * 1024, "tensor FIR shared memory exceeds the 227 KiB per-CTA limit");

// -DB2S_TC_TIMELINE (scripts/tc_timeline.py): every CTA writes %globaltimer stamps of the launch's edges, one thread per
// role, into g_tc_timeline[cta][TL_*]; b2s_tc_timeline_read copies them out.  The default build has none of it.
enum TcStamp { TL_ENTRY, TL_FIRST_COPY, TL_LAST_COPY, TL_FIRST_FULL, TL_FIRST_STORE, TL_LAST_STORE, TL_CONV_EXIT,
               TL_EXIT, TL_NSTAMPS };
#ifdef B2S_TC_TIMELINE
constexpr int kTlCtas = 1024;
__device__ unsigned long long g_tc_timeline[kTlCtas * TL_NSTAMPS];
#define TC_STAMP(k)                                                                          \
    do {                                                                                     \
        unsigned long long t_;                                                               \
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)::"memory");                     \
        if (blockIdx.x < kTlCtas) g_tc_timeline[blockIdx.x * TL_NSTAMPS + (k)] = t_;         \
    } while (0)
#else
#define TC_STAMP(k) do {} while (0)
#endif

// ---- PTX helpers ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
// one thread of a converged warp; unlike `lane == 0` the compiler knows exactly one thread is active, so
// uniform-datapath instructions (UBLKCP) are emitted bare instead of inside an ELECT retry loop
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Predicated global stores, branch-free in PTX: the epilogue needs no branches around its 32 stores, and ptxas
// serialises every wgmma of a kernel when registers are read on a path it must assume divergent between an mma_async
// and its wait_group.
__device__ __forceinline__ void st_global_if(float2 *p, float a, float b, bool pred) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %3, 0;\n\t@q st.global.v2.f32 [%0], {%1, %2};\n\t}"
                 ::"l"(p), "f"(a), "f"(b), "r"((int)pred) : "memory");
}
__device__ __forceinline__ void st_global_if(float *p, float a, bool pred) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t@q st.global.f32 [%0], %1;\n\t}"
                 ::"l"(p), "f"(a), "r"((int)pred) : "memory");
}
// per-thread register limit of the executing warpgroup (every warp of the warpgroup must execute the same one)
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// d[64] (+)= A[smem desc] * B[smem desc]   (m64n128k16, bf16 inputs, fp32 accumulate, both operands K-major)
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
        "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
        "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
// d[64] (+)= A[registers] * B[smem desc]: the A fragment of m64k16 as in mma.m16n8k16, one 16-row slice per warp
__device__ __forceinline__ void wgmma_m64n128_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc,
                                                 uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
        "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
        "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ uint32_t ld_shared_b32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

// f32 pair -> packed bf16x2 {lo16 = a, hi16 = b}, round-to-nearest-even (one XU instruction)
__device__ __forceinline__ uint32_t cvt_bf16x2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}
// split (a, b) into bf16 hi pair and bf16 lo pair:  x ~= hi + lo.
__device__ __forceinline__ void split2(float a, float b, uint32_t &hi, uint32_t &lo) {
    hi = cvt_bf16x2(a, b);
    const float ah = __uint_as_float(hi << 16), bh = __uint_as_float(hi & 0xffff0000u);
    lo = cvt_bf16x2(a - ah, b - bh);
}

// wgmma shared-memory matrix descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout [62,64)
// (0 = no swizzle, 1 = 128-byte swizzle)
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo, uint32_t layout) {
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32) |
           ((uint64_t)layout << 62);
}
// samples: K-major, SWIZZLE_128B, 8-row atoms 1024 B apart (LBO unused)
__device__ __forceinline__ uint64_t make_b_desc(uint32_t smem_addr) { return make_desc(smem_addr, 16, 1024, 1); }
// aliased Toeplitz taps: no swizzle, the next core matrix along K and along M is the same 128 bytes further
__device__ __forceinline__ uint64_t make_a_desc(uint32_t smem_addr) { return make_desc(smem_addr, 128, 128, 0); }

struct TcParams {
    const float *in;      // samples (float2 when COMPLEX)
    float *out;
    const float *g;       // g[t] = taps[N-1-t], t in [0, ntaps)
    long long n_in;       // items
    long long n_out;      // items
    int ntaps;
    int DK;               // K blocks of 128
    int num_tiles;
    int flags;            // tuning switches: bit1 skip the stores, bit2 skip the MMAs, bit3 skip the conversion
    int decim;            // D | 128: only the output phases p == D-1 (mod D) are stored (decimating FIR)
    // ---- misaligned / detached history (b2s_fir_exec_hist) -------------------------------------------------
    // The kernel's item coordinate i is:  [0, lead) dummy items that only exist to keep every bulk copy 16-byte
    // aligned (zeroed by the converters; the Toeplitz operand is shifted by `lead` columns so they meet zero
    // taps), [lead, hist_items) the detached history (`hist`, possibly PEER memory of the left-neighbour GPU,
    // fetched by the TMA loader over NVLink), [hist_items, n_in) the caller's slice.  `in` is the VIRTUAL base:
    // in + i addresses item i for i >= hist_items (hist_items == 0: everything is contiguous from `in`).
    const float *hist;    // 16-byte aligned address of item 0 when hist_items > 0
    int hist_items;       // lead + n_hist (a whole number of 16-byte units), 0 = contiguous input
    int lead;
    const unsigned *wait_flag;   // spin until *wait_flag >= wait_value (system scope) before reading hist
    unsigned wait_value;
    unsigned *done_flag;         // *done_flag = done_value (release, system scope) once hist sits in shared memory
    unsigned done_value;
    unsigned *pub_flag;          // *pub_flag = pub_value (release, system scope) as soon as the kernel runs: everything queued
    unsigned pub_value;          // before it on the stream (the chunk this rank owns) is in HBM
    unsigned *status;            // device status word of the context: bit0 = a flag wait timed out
    unsigned *sched;             // {next tile, CTAs done}: zero at launch, zero again when the last CTA is done
};

// ---------------------------------------------------------------------------------------------
// Tile = 128 columns = 16 swizzle atoms of 8 rows.
// COMPLEX: rows are (stream ri, block b); 64 blocks x 128 complex samples per tile, column
//          c = 8*gamma + 2*jb + ri  <->  block b0 + gamma + 16*jb   (gamma < 16, jb < 4)
// REAL   : 128 blocks x 128 samples per tile, column c = 8*gamma + j <-> block b0 + gamma + 16*j.
// In the wgmma accumulator layout a thread holds columns 8*gamma + 2*(lane%4) + {0,1}: the (re, im) pair of
// one complex output, or two real outputs 16 blocks apart.
// ---------------------------------------------------------------------------------------------
template <bool COMPLEX>
__global__ void __launch_bounds__(kThreadsTC, 1) fir_tc_kernel(const TcParams prm) {
    extern __shared__ unsigned char smem_raw[];
    // 1024-byte alignment for the 128B-swizzle atoms
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char *gen_base = smem_raw + (base - raw);
    const uint32_t raw_base = base + kStages * kStageBytes;           // raw f32 ring
    unsigned char *raw_gen = gen_base + kStages * kStageBytes;
    const uint32_t a_base = raw_base + kRawSlots * kRawSlotBytes;     // Toeplitz strip: hi, then lo
    __nv_bfloat16 *a_gen = reinterpret_cast<__nv_bfloat16 *>(raw_gen + kRawSlots * kRawSlotBytes);
    const uint32_t bar_base = a_base + 2 * kABytes;
    // barriers: full[kStages], empty[kStages], rfull[kRawSlots], rempty[kRawSlots]
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
    auto rfull_bar = [&](int r) { return bar_base + 8u * (2 * kStages + r); };
    auto rempty_bar = [&](int r) { return bar_base + 8u * (2 * kStages + kRawSlots + r); };
    // tile numbers handed down the pipeline (-1: no more tiles): loader -> converters per tile (ring of 4, indexed by
    // the CTA's tile count; the loader runs less than one tile ahead), converters -> math per operand stage
    const uint32_t tile_ring = bar_base + 8u * (2 * kStages + 2 * kRawSlots);
    const uint32_t stage_tile = tile_ring + 16u;
    volatile int *tile_ring_gen = reinterpret_cast<volatile int *>(gen_base + (tile_ring - base));
    volatile int *stage_tile_gen = reinterpret_cast<volatile int *>(gen_base + (stage_tile - base));

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) TC_STAMP(TL_ENTRY);
    if (prm.pub_flag && blockIdx.x == 0 && threadIdx.x == 0) {
        __threadfence_system();
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(prm.pub_flag), "r"(prm.pub_value) : "memory");
    }
    const int DK = prm.DK, K = 128 * DK;
    const int atoms = kAtomsOut + DK - 1;            // physical 8-row atoms per K-chunk
    const int chunk_bytes = atoms * 1024;            // one K-chunk (64 elements) of all rows
    const int split_bytes = 2 * chunk_bytes;
    constexpr int NSEQ = COMPLEX ? 4 : 8;            // interleaved block sub-sequences
    constexpr int TILE_BLOCKS = kAtomsOut * NSEQ;    // 64 / 128 blocks of 128 samples
    constexpr long long TILE_ITEMS = (long long)TILE_BLOCKS * 128;

    if (warp == kTmaWarp && lane == 0) {
        for (int s = 0; s < kStages; s++) { mbar_init(full_bar(s), kProdWarps); mbar_init(empty_bar(s), kMathWarps); }
        for (int r = 0; r < kRawSlots; r++) { mbar_init(rfull_bar(r), 1); mbar_init(rempty_bar(r), kProdWarps); }
        fence_barrier_init();
    }
    __syncthreads();                                 // barriers initialised: the loader starts streaming right away

    // ---- one-time, by the converters and the math warpgroups while the loader already streams: the aliased Toeplitz
    // strip.  Core matrix s, row r, element e (byte 128*s + 16*r + 2*e) holds A[p'][kappa] for every p' = 8a + r,
    // kappa = 8j + e with a + j = s:  g[kappa - p - lead], p = 127 - p' (`lead` zero taps in front meet the dummy
    // items).  Only the math warpgroups read it: the converters help build it and go on without waiting.
    auto build_strip = [&](auto wait_c) {
        const int a_elems = (K / 8 + 15) * 64;
        for (int i = threadIdx.x; i < a_elems; i += kNumMathThreads + kNumProducerThreads) {
            const int s = i >> 6, r = (i >> 3) & 7, e = i & 7;
            const int t = 8 * s + r + e - 127 - prm.lead;
            const float gv = (t >= 0 && t < prm.ntaps) ? __ldg(prm.g + t) : 0.0f;
            const __nv_bfloat16 hi = __float2bfloat16_rn(gv);
            a_gen[i] = hi;
            a_gen[kABytes / 2 + i] = __float2bfloat16_rn(gv - __bfloat162float(hi));
        }
        fence_proxy_async();                         // generic-proxy stores -> visible to wgmma (async proxy)
        if constexpr (decltype(wait_c)::value)       // named barrier 1: warps 0-15, never the loader
            asm volatile("bar.sync 1, %0;" ::"n"(kNumMathThreads + kNumProducerThreads) : "memory");
        else
            asm volatile("bar.arrive 1, %0;" ::"n"(kNumMathThreads + kNumProducerThreads) : "memory");
    };

    // A tile's contiguous input span (TILE_BLOCKS + DK - 1 blocks of 128 items) travels through the raw
    // ring in slots of 8 KiB = 512 float4 (8 complex blocks / 16 real blocks); 9 slots per tile.
    constexpr int F4_PER_BLOCK = COMPLEX ? 64 : 32;                       // float4 per 128-item block
    constexpr int BLOCKS_PER_SLOT = 512 / F4_PER_BLOCK;                   // 8 / 16
    constexpr int SLOTS_PER_TILE = (TILE_BLOCKS + kMaxDK - 1 + BLOCKS_PER_SLOT - 1) / BLOCKS_PER_SLOT;   // 9
    constexpr int ITEM_BYTES = COMPLEX ? 8 : 4;
    const int in_blocks = TILE_BLOCKS + DK - 1;

    if (warp >= kTmaWarp) {
        // ================================ TMA LOADER ===========================================
        // One thread streams the input with bulk async copies (cp.async.bulk): the copies complete on the
        // slot's mbarrier (complete_tx), so HBM latency is absorbed by the 48 KiB ring and never by a
        // converter warp's registers.
        // The CTA takes tiles from the launch's counter as its ring frees up, so an SM that streams faster takes more
        // tiles and all SMs run out of work within about one tile time of each other.
        setmaxnreg_dec<kLoaderRegs>();
        if (warp != kTmaWarp) return;
        if (elect_one()) {
            int rs = 0;
            uint32_t rphase = 0;
            for (int k = 0;; k++) {
                const int tile = (int)atomicAdd(prm.sched, 1u);
                if (tile >= prm.num_tiles) {
                    // no tile left: the end mark goes down the pipeline in place of a tile's first slot
                    mbar_wait(rempty_bar(rs), rphase ^ 1);
                    tile_ring_gen[k & 3] = -1;
                    mbar_arrive(rfull_bar(rs));
                    // the last CTA to find the counter spent zeroes it for the next launch on this slot
                    __threadfence();
                    if (atomicAdd(prm.sched + 1, 1u) == gridDim.x - 1) {
                        __threadfence();
                        atomicExch(prm.sched, 0u);
                        atomicExch(prm.sched + 1, 0u);
                    }
                    break;
                }
                tile_ring_gen[k & 3] = tile;          // published by the first slot's arrive (release)
                const long long item0 = (long long)tile * TILE_ITEMS;
#pragma unroll 1
                for (int s = 0; s < SLOTS_PER_TILE; s++) {
                    const int blk_first = s * BLOCKS_PER_SLOT;
                    if (blk_first >= in_blocks) break;
                    const int nblk = min(BLOCKS_PER_SLOT, in_blocks - blk_first);
                    const long long it0 = item0 + (long long)blk_first * 128;
                    long long items = (long long)nblk * 128;
                    if (it0 + items > prm.n_in) items = prm.n_in - it0;
                    long long bytes = items > 0 ? ((items * ITEM_BYTES) & ~15ll) : 0;    // whole 16-byte units
                    mbar_wait(rempty_bar(rs), rphase ^ 1);
                    if (tile == 0 && s == 0 && prm.hist_items > 0) {
                        // detached history: items [0, hist_items) come from `hist` (the left neighbour's tail over
                        // NVLink when it is peer memory), the rest of the slot from the caller's slice.
                        if (prm.wait_flag) {
                            unsigned long long t0, t1;
                            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
                            for (;;) {
                                unsigned v;
                                asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(prm.wait_flag) : "memory");
                                if ((int)(v - prm.wait_value) >= 0) break;
                                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
                                if (t1 - t0 > 4000000000ull) { atomicOr(prm.status, 1u); break; }   // 4 s: give up, flag it
                                __nanosleep(64);
                            }
                            asm volatile("fence.proxy.async;" ::: "memory");   // acquire (generic) -> bulk copy (async proxy)
                        }
                        const uint32_t hb = (uint32_t)prm.hist_items * ITEM_BYTES;
                        const uint32_t rest = bytes > (long long)hb ? (uint32_t)bytes - hb : 0u;
                        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(rfull_bar(rs)), "r"(hb + rest) : "memory");
                        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                     ::"r"(raw_base + rs * kRawSlotBytes), "l"(prm.hist), "r"(hb), "r"(rfull_bar(rs)) : "memory");
                        if (rest)
                            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                         ::"r"(raw_base + rs * kRawSlotBytes + hb), "l"(prm.in + (COMPLEX ? 2 : 1) * (long long)prm.hist_items),
                                           "r"(rest), "r"(rfull_bar(rs)) : "memory");
                    } else if (bytes > 0) {
                        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(rfull_bar(rs)), "r"((uint32_t)bytes) : "memory");
                        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                     ::"r"(raw_base + rs * kRawSlotBytes), "l"(prm.in + (COMPLEX ? 2 : 1) * it0),
                                       "r"((uint32_t)bytes), "r"(rfull_bar(rs)) : "memory");
                    } else {
                        mbar_arrive(rfull_bar(rs));          // nothing to copy (tile past the end): just hand it over
                    }
                    if (k == 0 && s == 0) TC_STAMP(TL_FIRST_COPY);
                    if (++rs == kRawSlots) { rs = 0; rphase ^= 1; }
                }
            }
            TC_STAMP(TL_LAST_COPY);
        }
        __syncwarp();
    } else if (warp >= kProdWarp0) {
        // ================================ CONVERTERS ===========================================
        // 256 threads; thread t owns float4 #t and #(t+256) of every raw slot.  Its position inside a
        // 128-item block (fo) and its row inside a slot (rowsel) never change, and the slot / float4
        // loops are fully unrolled, so every shared-memory address is
        //     stage base + per-thread constant + compile-time constant + one of 8 precomputed swizzle offsets.
        // Per float4: one LDS.128, two XU conversions per value pair, 4 (8 for aliased rows) 32-bit stores.
        build_strip(std::false_type{});
        setmaxnreg_dec<kProdRegs>();
        const int tid = threadIdx.x - 32 * kProdWarp0;                   // 0..255
        const int fo = tid % F4_PER_BLOCK, rowsel = tid / F4_PER_BLOCK;  // rowsel 0..3 (complex) / 0..7 (real)
        const int kc = COMPLEX ? (fo >> 5) : (fo >> 4);
        const int c16 = COMPLEX ? ((fo & 31) >> 2) : ((fo & 15) >> 1);
        const int wofs = COMPLEX ? (fo & 3) * 4 : (fo & 1) * 8;
        const uint32_t t_off = (uint32_t)(kc * chunk_bytes + wofs + rowsel * 1024);
        uint32_t xj[8];                                                   // row j: j*128 + ((c16 ^ j) << 4)
#pragma unroll
        for (int j = 0; j < 8; j++) xj[j] = (uint32_t)(j * 128 + ((c16 ^ j) << 4));
        const bool alias_thread = rowsel < DK - 1;                        // this thread's rows alias into atoms 16, 17
        const uint32_t sb = (uint32_t)split_bytes;

        // compile-time geometry of (slot s, float4 i): block bl = BLOCKS_PER_SLOT*s + rowsel + ROWS*i = gamma + 16*seq
        //   complex: gamma = 8*(s&1) + 4*i + rowsel, seq = s>>1 ;  real: gamma = 8*i + rowsel, seq = s
        auto convert_tile = [&](auto interior_c, unsigned char *stage_ptr, long long item0, int &rs, uint32_t &rphase) {
            constexpr bool INTERIOR = decltype(interior_c)::value;
            unsigned char *tp = stage_ptr + t_off;
#pragma unroll
            for (int s = 0; s < SLOTS_PER_TILE; s++) {
                if (s * BLOCKS_PER_SLOT >= in_blocks) break;
                mbar_wait(rfull_bar(rs), rphase);
                const float4 *raw = reinterpret_cast<const float4 *>(raw_gen + rs * kRawSlotBytes);
                float4 v[2];
                v[0] = raw[tid];
                v[1] = raw[tid + 256];
                const int rs_cur = rs;
                if (++rs == kRawSlots) { rs = 0; rphase ^= 1; }
                if constexpr (!INTERIOR) {
                    // the detached history has landed in shared memory: tell its owner it may be overwritten
                    if (s == 0 && item0 == 0 && tid == 0 && prm.done_flag)
                        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(prm.done_flag), "r"(prm.done_value) : "memory");
                }
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    constexpr int ROWS = COMPLEX ? 4 : 8;
                    const int g_ct = COMPLEX ? (8 * (s & 1) + 4 * i) : (8 * i);          // compile-time after unrolling
                    const int seq = COMPLEX ? (s >> 1) : s;
                    const bool alias_ct = COMPLEX ? ((s & 1) == 0 && i == 0 && s >= 2) : (i == 0 && s >= 1);
                    if (s == SLOTS_PER_TILE - 1) {                       // only the last slot can run past the tile's input
                        if (s * BLOCKS_PER_SLOT + rowsel + ROWS * i >= in_blocks) continue;
                    }
                    if (prm.flags & 8) continue;                         // tuning switch: skip conversion
                    if constexpr (!INTERIOR) {
                        // last tile: the bulk copy moved whole 16-byte units only; the <= 3 trailing floats are
                        // fetched directly, everything beyond the input is zero
                        const int bl = s * BLOCKS_PER_SLOT + rowsel + ROWS * i;
                        const long long it = item0 + (long long)bl * 128 + (long long)fo * (COMPLEX ? 2 : 4);
                        const long long gf = it * (COMPLEX ? 2 : 1);
                        const long long total_f = prm.n_in * (COMPLEX ? 2 : 1), copied_f = total_f & ~3ll;
                        float *e = reinterpret_cast<float *>(&v[i]);
                        const long long lead_f = (long long)prm.lead * (COMPLEX ? 2 : 1);
#pragma unroll
                        for (int c = 0; c < 4; c++) {
                            if (gf + c >= total_f || gf + c < lead_f) e[c] = 0.0f;
                            else if (gf + c >= copied_f) e[c] = prm.in[gf + c];
                        }
                    }
                    if constexpr (COMPLEX) {
                        uint32_t rh, rl, ih, il;                          // float4 = (re0, im0, re1, im1)
                        split2(v[i].x, v[i].z, rh, rl);
                        split2(v[i].y, v[i].w, ih, il);
                        if (seq < NSEQ) {
                            unsigned char *q = tp + g_ct * 1024;
                            *reinterpret_cast<uint32_t *>(q + xj[2 * (seq & 3)]) = rh;
                            *reinterpret_cast<uint32_t *>(q + xj[2 * (seq & 3)] + sb) = rl;
                            *reinterpret_cast<uint32_t *>(q + xj[2 * (seq & 3) + 1]) = ih;
                            *reinterpret_cast<uint32_t *>(q + xj[2 * (seq & 3) + 1] + sb) = il;
                        }
                        if (alias_ct && alias_thread) {                   // alias row (gamma+16, seq-1)
                            unsigned char *q = tp + (g_ct + kAtomsOut) * 1024;
                            *reinterpret_cast<uint32_t *>(q + xj[2 * ((seq - 1) & 3)]) = rh;
                            *reinterpret_cast<uint32_t *>(q + xj[2 * ((seq - 1) & 3)] + sb) = rl;
                            *reinterpret_cast<uint32_t *>(q + xj[2 * ((seq - 1) & 3) + 1]) = ih;
                            *reinterpret_cast<uint32_t *>(q + xj[2 * ((seq - 1) & 3) + 1] + sb) = il;
                        }
                    } else {
                        uint32_t h0, l0, h1, l1;                          // float4 = 4 consecutive samples
                        split2(v[i].x, v[i].y, h0, l0);
                        split2(v[i].z, v[i].w, h1, l1);
                        if (seq < NSEQ) {
                            unsigned char *q = tp + g_ct * 1024 + xj[seq & 7];
                            *reinterpret_cast<uint2 *>(q) = make_uint2(h0, h1);
                            *reinterpret_cast<uint2 *>(q + sb) = make_uint2(l0, l1);
                        }
                        if (alias_ct && alias_thread) {
                            unsigned char *q = tp + (g_ct + kAtomsOut) * 1024 + xj[(seq - 1) & 7];
                            *reinterpret_cast<uint2 *>(q) = make_uint2(h0, h1);
                            *reinterpret_cast<uint2 *>(q + sb) = make_uint2(l0, l1);
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(rempty_bar(rs_cur));          // values consumed: slot may be refilled
            }
        };

        int stage = 0, rs = 0;
        uint32_t phase = 0, rphase = 0;
        for (int k = 0;; k++) {
            mbar_wait(rfull_bar(rs), rphase);        // the tile's first slot, or the end mark
            const int tile = tile_ring_gen[k & 3];
            mbar_wait(empty_bar(stage), phase ^ 1);
            if (threadIdx.x == 32 * kProdWarp0) stage_tile_gen[stage] = tile;   // published by this warp's arrive
            if (tile < 0) {                          // no more tiles: pass the end mark on to the math warpgroups
                __syncwarp();
                if (lane == 0) mbar_arrive(full_bar(stage));
                break;
            }
            const long long item0 = (long long)tile * TILE_ITEMS;
            const bool interior = item0 + (long long)in_blocks * 128 <= prm.n_in &&
                                  !(tile == 0 && (prm.lead | prm.hist_items) != 0);   // tile 0 zeroes the dummy items
            unsigned char *stage_ptr = gen_base + stage * kStageBytes;
            if (interior) convert_tile(std::true_type{}, stage_ptr, item0, rs, rphase);
            else convert_tile(std::false_type{}, stage_ptr, item0, rs, rphase);
            fence_proxy_async();                     // generic-proxy stores -> visible to the MMA (async proxy)
            __syncwarp();
            if (lane == 0) mbar_arrive(full_bar(stage));
            if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
        if (threadIdx.x == 32 * kProdWarp0) TC_STAMP(TL_CONV_EXIT);
    } else {
        // ================================ MATH WARPGROUPS ======================================
        // Warpgroup wg computes the accumulator rows p' = 64*wg .. 64*wg+63 (output phases p = 127 - p') of
        // all 128 columns.  Thread (warp w, lane) holds rows 16*(w%4) + lane/4 + {0, 8} of its warpgroup and
        // columns 8*gamma + 2*(lane%4) + {0, 1}: acc[4*gamma + 2*h + e].
        build_strip(std::true_type{});
        setmaxnreg_inc<kMathRegs>();
        // warp-uniform by construction (a broadcast): the K-step loop below branches on it, and wgmma.mma_async in a
        // loop the compiler must assume divergent is serialised
        const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
        const int wl = warp & 3, q4 = lane & 3;
        // Decimation (decimating_fir.rs:80-92: o[k] = y[D-1 + k*D] of the full-rate FIR y): the MMAs still
        // produce every phase -- the kernel is HBM-bound below ~130 taps -- and the epilogue keeps the phases
        // p == D-1 (mod D).  D divides 128, so the kept phases are the same in every block and block b
        // contributes the 128/D outputs  k = b*(128/D) + (p-(D-1))/D.
        const int D = prm.decim, per_blk = 128 / D;
        const uint32_t a_hi = a_base + 1024u * wg, a_lo = a_hi + kABytes;   // row group a = 8*wg + a_local
        // The warpgroup's phases p in [p0, p0 + 63] meet taps only in the Toeplitz columns
        // kappa in [p0 + lead, p0 + 63 + lead + ntaps - 1]: K-steps j (kappa = 16j .. 16j+15) outside [j0, j0 + nsteps) would
        // add only zero products and are not issued.  flags bit2 (tuning switch): no MMAs at all.
        const int p0 = 64 * (1 - wg);
        const int j0 = p0 / 16;                      // = (p0 + lead) / 16, lead < 16; a multiple of 4
        const int nsteps = (prm.flags & 4) ? 0 : min((p0 + 63 + prm.lead + prm.ntaps - 1) / 16, 8 * DK - 1) - j0 + 1;

        // g_hi feeds two of the three products of every K-step, so it is held in registers for the whole kernel (RS
        // wgmma) instead of being read from shared memory by both MMAs of every K-step of every tile.  Fragment i
        // (K-step j0 + i) of warp wl: rows 16*wl + lane/4 + {0, 8}, K pairs 2*(lane%4) + {0, 8}, i.e. the 32-bit word
        // at row lane/4, element 2*(lane%4) of the strip's core matrices s, s + 1, s + 1, s + 2 (rows + 8 and K + 8
        // are the same core matrix of the aliased strip), s = 8*wg + 2*wl + 2*j.  Loaded once; a fragment register is
        // never written again, so no MMA in flight can see it change.
        uint32_t ghi[kMaxKSteps][4];
        {
            const uint32_t f0 = a_hi + 256u * (uint32_t)(wl + j0) + 16u * (uint32_t)(lane >> 2) + 4u * (uint32_t)q4;
#pragma unroll
            for (int i = 0; i < kMaxKSteps; i++) {
                const uint32_t f = f0 + 256u * i;
                const bool used = i < nsteps;
                ghi[i][0] = used ? ld_shared_b32(f) : 0u;
                ghi[i][1] = used ? ld_shared_b32(f + 128u) : 0u;
                ghi[i][2] = used ? ld_shared_b32(f + 128u) : 0u;
                ghi[i][3] = used ? ld_shared_b32(f + 256u) : 0u;
            }
        }

        const uint64_t a_lo_desc = make_a_desc(a_lo + 256u * j0);   // K-step j reads core matrices a + 2j, a + 2j + 1

        int stage = 0;
        uint32_t phase = 0;
        // issue the full stage's MMAs into acc and commit them
        auto mma_tile = [&](float (&acc)[64]) {
            wgmma_fence();                           // earlier register reads of acc precede the async writes
            // Shared-memory addresses stay below 2^18, so a byte offset moves a descriptor's start field by offset / 16
            // without a carry: the per-K-step descriptors are the tile's base descriptors plus small offsets.
            const uint64_t b_desc = make_b_desc(base + stage * kStageBytes);
#pragma unroll
            for (int i = 0; i < kMaxKSteps; i++) {   // unrolled: the fragment index must be static
                if (i >= nsteps) break;
                const int m = (j0 >> 2) + (i >> 2);  // K-step j = j0 + i: d = m >> 1, kc = m & 1, ks = i & 3
                const uint64_t bh = b_desc + (uint32_t)(((m & 1) * chunk_bytes + (m >> 1) * 1024 + (i & 3) * 32) >> 4);
                wgmma_m64n128_rs(acc, ghi[i], bh, i != 0);                                // g_hi * x_hi
                wgmma_m64n128_rs(acc, ghi[i], bh + (uint32_t)(split_bytes >> 4), 1u);     // g_hi * x_lo
                wgmma_m64n128(acc, a_lo_desc + 16u * i, bh, 1u);                          // g_lo * x_hi
            }
            wgmma_commit();
        };
        // wait for the MMAs, then hand the operand stage back to the converters (they may refill it)
        auto release_stage = [&]() {
            wgmma_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(stage));
            if (++stage == kStages) { stage = 0; phase ^= 1; }
        };
        // ---- epilogue: for each (h, gamma) a warp writes 4 runs of 8 consecutive outputs (one per lane%4).  The
        // output of column gamma is kb + gamma * per_blk (+ 16 * per_blk for the second real value); it is written when
        // its phase is kept and k < n_out, i.e. gamma * per_blk < room, i.e. gamma < ncols.  D is a power of two
        // (D | 128), and so is per_blk.
        const int log2D = __ffs(D) - 1;
        auto store_tile = [&](const float (&acc)[64], int tile) {
            if (prm.flags & 2) return;                      // tuning switch: skip the global stores
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int p = 127 - (64 * wg + 16 * wl + (lane >> 2) + 8 * h);
                const int keep = (p & (D - 1)) == D - 1;
                const long long kb = ((long long)tile * TILE_BLOCKS + kAtomsOut * q4 * (COMPLEX ? 1 : 2)) * per_blk +
                                     (p >> log2D);
                const int room = (int)max(min(prm.n_out - kb, (long long)INT_MAX), 0ll) & -keep;
                const int ncols = (int)(((unsigned)room + (unsigned)per_blk - 1u) >> (7 - log2D));   // ceil(room / per_blk)
                if constexpr (COMPLEX) {
#pragma unroll
                    for (int gam = 0; gam < 16; gam++)
                        st_global_if(reinterpret_cast<float2 *>(prm.out) + kb + gam * per_blk, acc[4 * gam + 2 * h],
                                     acc[4 * gam + 2 * h + 1], gam < ncols);
                } else {
                    // the two values of column gamma are outputs gamma and gamma + 16 of one run of 32, per_blk apart:
                    // one address stream, and predicates against constants, keep the epilogue inside the math
                    // warpgroups' registers next to the g_hi fragments
#pragma unroll
                    for (int n = 0; n < 2 * kAtomsOut; n++)
                        st_global_if(prm.out + (kb + n * per_blk), acc[4 * (n % kAtomsOut) + 2 * h + n / kAtomsOut],
                                     n < ncols);
                }
            }
        };

        // One accumulator set: the g_hi fragments take the registers a second set would need, so a tile is stored
        // after its MMAs completed (the converters keep filling the other operand stage meanwhile).
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; i++) acc[i] = 0.0f;
        for (int k = 0;; k++) {
            mbar_wait(full_bar(stage), phase);
            // the stage's tile, or the end mark; a broadcast, so that the loop is warp-uniform by construction
            const int tile = __shfl_sync(0xffffffffu, stage_tile_gen[stage], 0);
            if (tile < 0) break;
            mma_tile(acc);
            if (threadIdx.x == 0 && k == 0) TC_STAMP(TL_FIRST_FULL);   // (+ its MMAs issued)
            release_stage();
            if (threadIdx.x == 0) TC_STAMP(TL_LAST_STORE);            // (overwritten until the last tile)
            store_tile(acc, tile);
            if (threadIdx.x == 0 && k == 0) TC_STAMP(TL_FIRST_STORE);
        }
        if (threadIdx.x == 0) TC_STAMP(TL_EXIT);
    }
}

}  // namespace

bool fir_tc_supported(const b2s_fir *f) {
    if (f->decim == 0 || f->decim > 128 || 128 % f->decim != 0) return false;   // kept output phases must be lane-static
    if (f->kind != B2S_C32_F32 && f->kind != B2S_F32_F32) return false;
    // >= 16 taps: with fewer products the split-bf16 error (O(2^-17) per product) no longer averages
    // below the 1e-5 * ||taps||_1 * max|x| bar; short filters are HBM-bound on CUDA cores anyway.
    return f->ntaps >= 16 && f->ntaps <= 128 * kMaxDK - 127;   // K = 128*DK >= ntaps + 127
}

int32_t fir_tc_prepare(b2s_fir *f) {
    b2s_ctx *ctx = f->ctx;
    if (f->tc_ready) return B2S_OK;
    if (!fir_tc_supported(f)) return b2s_fail(ctx, B2S_EUNSUPPORTED, "tensor FIR: unsupported plan");
    // g[t] = taps[N-1-t] already sits behind the phase table of the direct plan (fir_direct_prepare)
    f->tc_kblocks = (int)ceil_div(f->ntaps + 127, 128);
    B2S_CUDA(ctx, cudaFuncSetAttribute(fir_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTC));
    B2S_CUDA(ctx, cudaFuncSetAttribute(fir_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTC));
    // the setmaxnreg budget holds only for the entry register count it was sized for; any other would hang the kernel
    for (const void *k : {(const void *)fir_tc_kernel<true>, (const void *)fir_tc_kernel<false>}) {
        cudaFuncAttributes attr;
        B2S_CUDA(ctx, cudaFuncGetAttributes(&attr, k));
        if (attr.numRegs != kRegsAtLaunch)
            return b2s_fail(ctx, B2S_EUNSUPPORTED, "tensor FIR: kernel built with %d registers per thread, its setmaxnreg "
                            "budget assumes %d", attr.numRegs, kRegsAtLaunch);
    }
    if (const char *e = getenv("B2S_TC_FLAGS")) f->tc_flags = atoi(e);
    B2S_TRY(f->d_tc_sched.alloc(ctx, 2 * kSchedSlots, "tensor FIR: tile counters"));
    B2S_CUDA(ctx, cudaMemset(f->d_tc_sched.get(), 0, 2 * kSchedSlots * sizeof(unsigned)));
    f->tc_ready = true;
    return B2S_OK;
}

// The tensor kernel moves its input with 16-byte bulk copies.  A slice that starts on an item boundary but not on a
// 16-byte one (a ring slot's [halo | chunk] with 255 items of history, say) is handled by starting `lead` items
// early and shifting the Toeplitz operand by `lead` zero taps; a DETACHED history (hist, possibly peer memory) is
// fetched by the loader in front of tile 0.  Returns B2S_EAGAIN when this call cannot run on the tensor kernel
// (the caller then copies the history in place and/or uses the CUDA-core kernel).
int32_t fir_tc_launch_hist(b2s_fir *f, const FirHist *h, const void *d_in, size_t n_in, void *d_out, size_t n_out,
                           cudaStream_t stream) {
    b2s_ctx *ctx = f->ctx;
    if (n_out == 0) return B2S_OK;
    if (!f->tc_ready) return b2s_fail(ctx, B2S_ESTATE, "tensor FIR not prepared");
    const bool cplx = f->kind == B2S_C32_F32;
    const size_t item = cplx ? 8 : 4, q = 16 / item;
    const uintptr_t a_in = reinterpret_cast<uintptr_t>(d_in), a_out = reinterpret_cast<uintptr_t>(d_out);
    if ((a_in % item) || (a_out % item)) return B2S_EAGAIN;
    const size_t n_hist = h ? h->n_hist : 0;
    size_t lead;
    if (n_hist) {
        const uintptr_t a_h = reinterpret_cast<uintptr_t>(h->d_hist);
        if ((a_h % item) || (a_in & 15)) return B2S_EAGAIN;
        lead = (a_h / item) % q;
        if ((lead + n_hist) % q) return B2S_EAGAIN;
        if (lead + n_hist > 1024 || n_in * item < 16) return B2S_EAGAIN;     // must fit the first raw slot
    } else {
        lead = (a_in / item) % q;
    }
    const int DK = (int)ceil_div(f->ntaps + lead + 127, 128);
    if (DK > kMaxDK) return B2S_EAGAIN;
    TcParams prm;
    prm.lead = (int)lead;
    prm.hist_items = n_hist ? (int)(lead + n_hist) : 0;
    prm.hist = n_hist ? (const float *)h->d_hist - lead * (item / 4) : nullptr;
    // virtual base: item i of the kernel's coordinate lives at in + i for i >= hist_items
    prm.in = (const float *)d_in - (lead + n_hist) * (item / 4);
    prm.wait_flag = (h && n_hist) ? h->wait_flag : nullptr;
    prm.wait_value = h ? h->wait_value : 0;
    prm.done_flag = (h && n_hist) ? h->done_flag : nullptr;
    prm.done_value = h ? h->done_value : 0;
    prm.pub_flag = h ? h->publish_flag : nullptr;
    prm.pub_value = h ? h->publish_value : 0;
    prm.status = ctx->d_status;
    // a launch's tile counter: one of kSchedSlots per plan in turn, so launches of the plan in flight at the same time
    // (on different streams) use different counters
    prm.sched = f->d_tc_sched.get() + 2 * (f->tc_launches++ % kSchedSlots);
    prm.out = (float *)d_out;
    prm.g = f->d_ptaps.get() + (size_t)f->decim * f->Upad;      // plain reversed taps (fir_direct_prepare)
    prm.n_in = (long long)(lead + n_hist + n_in);
    prm.n_out = (long long)n_out;                        // decimated count
    prm.decim = (int)f->decim;
    prm.ntaps = (int)f->ntaps;
    prm.DK = DK;
    const long long tile_items = cplx ? 64 * 128 : 128 * 128;
    prm.num_tiles = (int)ceil_div(n_out * f->decim, (size_t)tile_items);   // tiles over the full-rate index space
    prm.flags = f->tc_flags;
    const int grid = std::min(prm.num_tiles, ctx->sm_count);
    if (prm.wait_flag) ctx->flag_ops++;
    if (cplx) fir_tc_kernel<true><<<grid, kThreadsTC, kSmemTC, stream>>>(prm);
    else fir_tc_kernel<false><<<grid, kThreadsTC, kSmemTC, stream>>>(prm);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

#ifdef B2S_TC_TIMELINE
// Copies the stamps of the most recent launch for CTAs [0, ctas) into host[cta * TL_NSTAMPS + stamp] (nanoseconds,
// %globaltimer) and clears them; returns TL_NSTAMPS, or -1 on a CUDA error.  Synchronous.
extern "C" int b2s_tc_timeline_read(unsigned long long *host, int ctas) {
    const size_t bytes = sizeof(unsigned long long) * TL_NSTAMPS * (size_t)std::min(std::max(ctas, 0), kTlCtas);
    void *d = nullptr;
    if (cudaGetSymbolAddress(&d, g_tc_timeline) != cudaSuccess) return -1;
    if (cudaMemcpy(host, d, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    if (cudaMemset(d, 0, sizeof(unsigned long long) * TL_NSTAMPS * kTlCtas) != cudaSuccess) return -1;
    return TL_NSTAMPS;
}
#endif

int32_t fir_tc_launch(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out,
                      cudaStream_t stream) {
    const int32_t rc = fir_tc_launch_hist(f, nullptr, d_in, n_in, d_out, n_out, stream);
    if (rc == B2S_EAGAIN) return fir_direct_launch(f, d_in, n_in, d_out, n_out, stream);   // item-misaligned slices
    return rc;
}
