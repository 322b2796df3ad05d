// tx_common.cuh -- the host-side bookkeeping the device transmitters share (lora.cu, wlan.cu): device rings that grow
// on push, and the queue of frames not yet fully produced with its burst_start records.
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
