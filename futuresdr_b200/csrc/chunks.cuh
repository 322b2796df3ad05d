// chunks.cuh -- the aligned-chunk loop of the element-wise streaming kernels (stream.cu, sigsrc.cu), and the launch
// geometry they share with the per-item grid-stride kernels (apply.cu, rotator.cu).
//
// Slices are item-aligned only (4 bytes is enough), and the streams of one call may be misaligned differently, so
// items are moved as 32-bit words.  A call of m items is cut into
//   * a scalar head of `head` items (0..3, head_items() on the host), which brings one chosen stream to 16 bytes;
//   * (m - head) / 4 chunks of 4 items, walked grid-stride; every stream whose chunks are then 16-byte aligned is
//     moved with float4 accesses (ld_chunk / st_chunk with wide = aligned16(..)), the others word by word;
//   * a scalar tail of the (m - head) % 4 items left.
// Any offset and length works, 0 and 1 included.  The head and tail items go to the first threads of the grid:
// thread g < head takes item g, thread head + k takes tail item k.
#pragma once

#include <algorithm>
#include <cstdint>

#include "common.cuh"

constexpr int kThreads = 256;       // threads per CTA
constexpr int kBlocksPerSm = 8;     // CTAs per SM that a grid-stride grid asks for

// ---- 4-item chunks of W-word items ---------------------------------------------------------------------------
template <int W> __device__ __forceinline__ void ld_chunk(const float *__restrict__ p, bool wide, float (&r)[4 * W]) {
    if (wide) {
#pragma unroll
        for (int j = 0; j < W; j++) {
            const float4 q = __ldg(reinterpret_cast<const float4 *>(p) + j);
            r[4 * j] = q.x; r[4 * j + 1] = q.y; r[4 * j + 2] = q.z; r[4 * j + 3] = q.w;
        }
    } else {
#pragma unroll
        for (int j = 0; j < 4 * W; j++) r[j] = __ldg(p + j);
    }
}

template <int W> __device__ __forceinline__ void st_chunk(float *__restrict__ p, bool wide, const float (&r)[4 * W]) {
    if (wide) {
#pragma unroll
        for (int j = 0; j < W; j++)
            reinterpret_cast<float4 *>(p)[j] = make_float4(r[4 * j], r[4 * j + 1], r[4 * j + 2], r[4 * j + 3]);
    } else {
#pragma unroll
        for (int j = 0; j < 4 * W; j++) p[j] = r[j];
    }
}

__device__ __forceinline__ bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// This thread's share of m items (head <= m, a grid of kThreads-thread CTAs): chunk(v) for every chunk v it owns
// (items head + 4 v .. head + 4 v + 3), then item(i) for at most one head or tail item i.
template <class Chunk, class Item>
__device__ __forceinline__ void chunk_loop(unsigned long long m, unsigned head, Chunk chunk, Item item) {
    const unsigned long long g = (unsigned long long)blockIdx.x * kThreads + threadIdx.x;
    const unsigned long long nv = (m - head) >> 2;
    for (unsigned long long v = g; v < nv; v += (unsigned long long)gridDim.x * kThreads) chunk(v);
    const unsigned long long tail0 = head + 4 * nv;
    unsigned long long i = ~0ull;
    if (g < head) i = g;
    else if (g - head < m - tail0) i = tail0 + (g - head);
    if (i != ~0ull) item(i);
}

// first item count (0..3) that brings `addr` to 16 bytes, 0 if no count does
static inline unsigned head_items(const void *addr, size_t item_bytes) {
    for (unsigned h = 0; h < 4; h++)
        if ((((uintptr_t)addr + h * item_bytes) & 15) == 0) return h;
    return 0;
}

// CTAs of kThreads threads for `units` units of work (chunks or items), at most per_sm per SM and at least one
static inline unsigned grid_for(b2s_ctx *ctx, unsigned long long units, int per_sm = kBlocksPerSm) {
    return (unsigned)std::max<unsigned long long>(
        1, std::min<unsigned long long>(ceil_div(units, (size_t)kThreads), (unsigned long long)ctx->sm_count * per_sm));
}
