// tx_common.cuh -- what the device transmitters share (lora.cu, wlan.cu, zigbee_tx.cu): device rings that grow on push,
// the queue of frames not yet fully produced with its burst_start records, and the exec kernels' frame search and
// streaming stores.
#pragma once

#include <algorithm>
#include <deque>
#include <vector>

#include "common.cuh"

// Items are numbered by absolute counters; item a lives at a & (capacity - 1).  Growing moves the live items
// [tail, head) to the new capacity under the same numbers, and synchronises.
template <typename T> struct DevRing {
    Buf<T> b;
    unsigned long long mask() const { return b.size() ? b.size() - 1 : 0; }
    int32_t make_room(b2s_ctx *ctx, unsigned long long tail, unsigned long long head, size_t n, const char *what) {
        const size_t live = head - tail;
        if (live + n <= b.size()) return B2S_OK;
        size_t cap = b.size() ? b.size() : 1024;
        while (cap < live + n) cap *= 2;
        Buf<T> nb;
        B2S_TRY(nb.alloc(ctx, cap, what));
        for (unsigned long long a = tail; a < head;) {
            const size_t so = a & mask(), d = a & (cap - 1);
            const size_t k = std::min<size_t>({head - a, b.size() - so, cap - d});
            B2S_CUDA(ctx, cudaMemcpyAsync(nb.get() + d, b.get() + so, k * sizeof(T), cudaMemcpyDeviceToDevice,
                                          ctx->stream));
            a += k;
        }
        B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        b = std::move(nb);
        return B2S_OK;
    }
    // n host items to positions [a, a + n)
    int32_t put(b2s_ctx *ctx, unsigned long long a, const T *host, size_t n) {
        for (size_t i = 0; i < n;) {
            const size_t d = (a + i) & mask(), k = std::min(n - i, b.size() - d);
            B2S_CUDA(ctx, cudaMemcpyAsync(b.get() + d, host + i, k * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
            i += k;
        }
        return B2S_OK;
    }
};

// One queued frame: stream index of its first sample, its samples, its first symbol in the symbol ring.
struct TxHostFrame {
    unsigned long long start, len, sym_abs;
};

// The frames of a transmitter between push and the exec that produces their last sample.  Frame f_tail is the front
// of `queue`; frames and symbols are numbered as in the device rings.  Burst is a {index, len} record of the header.
template <typename Burst> struct TxQueue {
    std::deque<TxHostFrame> queue;
    unsigned long long f_tail = 0, f_head = 0, s_tail = 0, s_head = 0;
    unsigned long long pos = 0, total = 0;   // samples produced, samples queued
    bool finishing = false;
    std::vector<Burst> bursts;
    size_t bursts_rd = 0;

    void reset() {
        queue.clear();
        f_tail = f_head;
        s_tail = s_head;
        pos = total = 0;
        finishing = false;
        bursts.clear();
        bursts_rd = 0;
    }
    // frames pushed after the queued ones: hf[i].start continues the stream, n_sym symbols after s_head
    void append(const std::vector<TxHostFrame> &hf, unsigned long long n_sym) {
        queue.insert(queue.end(), hf.begin(), hf.end());
        f_head += hf.size();
        s_head += n_sym;
        if (!hf.empty()) total = hf.back().start + hf.back().len;
    }
    // the frames that samples [pos, end) touch, from f_tail on; records the burst of each frame that starts there
    size_t open(unsigned long long end) {
        size_t n = 0;
        for (const TxHostFrame &f : queue) {
            if (f.start >= end) break;
            if (f.start >= pos) bursts.push_back(Burst{f.start, f.len});   // burst_start tag
            ++n;
        }
        return n;
    }
    // samples up to `end` are produced: drop the frames that ended
    void close(unsigned long long end) {
        pos = end;
        while (!queue.empty() && queue.front().start + queue.front().len <= pos) {
            queue.pop_front();
            ++f_tail;
        }
        s_tail = queue.empty() ? s_head : queue.front().sym_abs;
    }
    bool finished() const { return finishing && pos == total; }
    size_t drain(Burst *host, size_t cap) {
        const size_t k = std::min(cap, bursts.size() - bursts_rd);
        std::copy(bursts.begin() + bursts_rd, bursts.begin() + bursts_rd + k, host);
        bursts_rd += k;
        if (bursts_rd == bursts.size()) {
            bursts.clear();
            bursts_rd = 0;
        }
        return k;
    }
};

// The last of the n frame records frames[(f_lo + i) & mask], i < n, ascending in .start, whose start is at or before t:
// a 32-ary search by one whole warp; every lane returns the index i.
template <typename Rec>
__device__ __forceinline__ unsigned long long tx_first_frame(const Rec *frames, unsigned long long mask,
                                                             unsigned long long f_lo, unsigned long long n,
                                                             unsigned long long t) {
    const unsigned lane = threadIdx.x & 31;
    unsigned long long lo = 0;
    while (n > 1) {
        const unsigned long long step = (n + 31) / 32, i = lo + lane * step;
        const bool le = lane * step < n && frames[(f_lo + i) & mask].start <= t;
        const unsigned bal = __ballot_sync(~0u, le);
        const unsigned last = bal ? 31 - __clz(bal) : 0;
        lo += last * step;
        n = min(step, n - last * step);
    }
    return lo;
}

// dst[i] = f(i) for i in [i0, i1) by the CTA's Threads threads, two samples per 16-byte streaming store where dst + i
// is 16-byte aligned (the output is only 8-byte aligned)
template <int Threads, typename I, typename F>
__device__ __forceinline__ void store_range(float2 *dst, I i0, I i1, F f) {
    if (i0 >= i1) return;
    if ((reinterpret_cast<uintptr_t>(dst + i0) & 15) != 0) {
        if (threadIdx.x == 0) __stcs(dst + i0, f(i0));
        ++i0;
    }
    const I n2 = (i1 - i0) / 2;
    for (I p = threadIdx.x; p < n2; p += Threads) {
        const I i = i0 + 2 * p;
        const float2 v0 = f(i), v1 = f(i + 1);
        __stcs(reinterpret_cast<float4 *>(dst + i), make_float4(v0.x, v0.y, v1.x, v1.y));
    }
    if (((i1 - i0) & 1) && threadIdx.x == Threads - 1) __stcs(dst + i1 - 1, f(i1 - 1));
}
