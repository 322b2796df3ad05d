// lists.cuh -- the result lists of the blocks that turn a stream into messages (ADS-B packets and detections, ZigBee
// frames).  A list lives in device memory and its length in the block's device state; kernels append to it in stream
// order.  The host never waits for a count to launch an exec: it keeps an upper bound of each length, grows a list only
// when an exec's worst case no longer fits, and tightens the bounds to the true lengths once a copy of them, made
// behind an earlier exec, has landed in pinned memory.  Draining synchronises.
#pragma once

#include <algorithm>
#include <initializer_list>
#include <vector>

#include "common.cuh"

// a list that keeps its first `valid` entries when it grows (stream-ordered copy, then the old memory is freed)
template <typename T> int32_t list_grow(b2s_ctx *ctx, Buf<T> &b, size_t need, size_t valid, const char *what) {
    if (b.size() >= need) return B2S_OK;
    Buf<T> nb;
    B2S_TRY(nb.alloc(ctx, std::max<size_t>({need, 2 * b.size(), 1024}), what));
    valid = std::min(valid, b.size());
    if (valid) B2S_CUDA(ctx, cudaMemcpyAsync(nb.get(), b.get(), valid * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    b = std::move(nb);
    return B2S_OK;
}

// The lengths of a block's N lists, copied to pinned memory behind its last exec.  Once `landed` has completed the
// host takes them as exact bounds, so an undrained block's lists grow with what it found, not with the worst case.
template <int N> struct ListCounts {
    Buf<unsigned long long, Mem::Pinned> host;
    cudaEvent_t landed = nullptr;
    bool pending = false;
    ListCounts() = default;
    ListCounts(const ListCounts &) = delete;
    ListCounts &operator=(const ListCounts &) = delete;
    ~ListCounts() {
        if (landed) cudaEventDestroy(landed);
    }
    int32_t init(b2s_ctx *ctx, const char *what) {
        B2S_TRY(host.alloc(ctx, N, what));
        B2S_CUDA(ctx, cudaEventCreateWithFlags(&landed, cudaEventDisableTiming));
        return B2S_OK;
    }
    // the copy behind the last exec: if it has landed (waiting for it first when `wait`), bounds[i] = count i
    int32_t refresh(b2s_ctx *ctx, bool wait, std::initializer_list<size_t *> bounds) {
        if (pending && wait) B2S_CUDA(ctx, cudaEventSynchronize(landed));
        if (!pending) return B2S_OK;
        const cudaError_t q = cudaEventQuery(landed);
        if (q == cudaSuccess) {
            int i = 0;
            for (size_t *b : bounds) *b = (size_t)host.get()[i++];
            pending = false;
        } else if (q == cudaErrorNotReady) {
            cudaGetLastError();                              // not an error: the last exec is still running
        } else {
            B2S_CUDA(ctx, q);
        }
        return B2S_OK;
    }
    // copy N consecutive device counts from d_counts behind the work queued so far
    int32_t record(b2s_ctx *ctx, const unsigned long long *d_counts) {
        B2S_CUDA(ctx, cudaMemcpyAsync(host.get(), d_counts, N * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                                      ctx->stream));
        B2S_CUDA(ctx, cudaEventRecord(landed, ctx->stream));
        pending = true;
        return B2S_OK;
    }
};

// Copy up to cap entries [rd, count) of `list` to `host` (keeping those `keep` accepts), and empty the list once all
// are out.  `d_cnt` is the list's length in device memory; the drain leaves `bound` exact.
template <typename T, typename H, int N, class K>
int32_t list_drain(b2s_ctx *ctx, Buf<T> &list, unsigned long long *d_cnt, ListCounts<N> &counts, size_t &rd,
                   size_t &bound, H *host, size_t cap, size_t *n, K keep) {
    DeviceGuard g(ctx->device);
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    unsigned long long cnt = 0;
    B2S_CUDA(ctx, cudaMemcpy(&cnt, d_cnt, sizeof(cnt), cudaMemcpyDeviceToHost));
    size_t out = 0;
    std::vector<T> tmp;
    while (out < cap && rd < cnt) {
        const size_t k = std::min<size_t>(cap - out, cnt - rd);
        tmp.resize(k);
        B2S_CUDA(ctx, cudaMemcpy(tmp.data(), list.get() + rd, k * sizeof(T), cudaMemcpyDeviceToHost));
        for (const T &e : tmp)
            if (keep(e)) std::memcpy(host + out++, &e, sizeof(T));
        rd += k;
    }
    counts.pending = false;                     // the bounds below are exact
    if (rd == cnt) {
        const unsigned long long zero = 0;
        B2S_CUDA(ctx, cudaMemcpy(d_cnt, &zero, sizeof(zero), cudaMemcpyHostToDevice));
        rd = 0;
        bound = 0;
    } else {
        bound = cnt;
    }
    *n = out;
    return B2S_OK;
}
