// keyfob.cu -- the keyfob receiver's Decoder (examples/keyfob/src/decoder.rs:64-127, with print at :36-52) as a device
// block (DESIGN §4.17).  With the resampler, Apply(NormSqr), Apply(DcBlockF32), the FIR and Apply(SliceF32U8) in front
// it is the receive chain of examples/keyfob/src/main.rs:39-79, and only the decoded key codes leave the device.
//
// The decoder is a walk over edges (a 1 while Down, a 0 while Up; every other item is ignored) whose decisions are all
// scans with bounded state, so no step is serial in edges:
//   1. tile_summary   per tile of 4096 items (16-byte loads): the last binary item, the first binary item and the last
//                     edge that does not depend on the level the tile is entered with.
//   2. tile_scan      one CTA: two max-scans over the tiles give each tile its entry level and its incoming `since`.
//   3. tile_events    per tile again: every edge gets its class from `diff = pos - since` (63..=83 short, 131..=161
//                     long, otherwise a flush).  Short and long edges are kept as events, and of the flushes only the
//                     first of the tile and those right after a short or long edge: a flush that follows a flush
//                     finds the string empty and does nothing.  Short / long edges are at least 63 items apart, so a
//                     tile keeps at most 133 events.
//   4. walk_kernel    one warp over the kept events, 32 at a time: the output flag as a scan of {toggle, 0, identity},
//                     then the appended bits as a ballot, an 8-bit match of 10101111 over a 64-bit window, and the
//                     reports.  Its work grows with the appended bits (and one event per tile), not with the edges.
#include <cstdint>

#include "lists.cuh"

namespace {

constexpr int kTileThreads = 256;
constexpr int kPerThread = 16;                          // one 16-byte vector of u8 items
constexpr int kTile = kTileThreads * kPerThread;        // 4096 items
constexpr int kEvCap = 136;                             // events a tile can keep (<= 66 short/long + 67 flushes)
constexpr int kScanThreads = 1024;
constexpr unsigned long long kNone = ~0ull;
constexpr unsigned kPreamble = 0xAFu;                   // "10101111", the first bit in bit 7

enum Kind : unsigned { kShort = 0, kLong = 1, kFlush = 2 };

struct Code {                                           // == b2s_keyfob_code
    unsigned long long index;
    unsigned n_bits;
    int label;
    unsigned char bits[32];
};
static_assert(sizeof(Code) == sizeof(b2s_keyfob_code), "ABI layout");

struct KfState {
    unsigned long long pos0;        // stream index of the slice start
    unsigned long long since;       // State::{Up,Down}(since)
    unsigned long long n_codes;     // codes in the list
    unsigned long long str_len;     // output_string.len()
    unsigned long long pre;         // string index of the first 10101111, kNone if there is none yet
    unsigned level;                 // 1 = Up, 0 = Down
    unsigned flag;                  // `output`
    unsigned last32;                // the string's last 32 bits, the newest in bit 0
    unsigned pad;
    unsigned cap[8];                // the string's bits from `pre` (at most 256), MSB first per byte
};

struct TileRec {
    unsigned long long last_bin;    // ((rel + 1) << 1) | value of the tile's last binary item, 0 if none
    unsigned long long first_bin;   // (rel << 1) | value of its first binary item, kNone if none
    unsigned long long local_edge;  // rel + 1 of its last edge that does not depend on the entry level, 0 if none
};

// ---- block scans (max or sum over u64) ----------------------------------------------------------------------------
struct Max { __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a > b ? a : b; } };
struct Sum { __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a + b; } };

// exclusive scan of v over the CTA (thread order), seeded with `init`; *total = init op (all v).  sh: NT/32 + 1 words.
template <int NT, class Op>
__device__ unsigned long long block_excl(unsigned long long v, unsigned long long init, Op op, unsigned long long *sh,
                                         unsigned long long *total) {
    constexpr int kW = NT / 32;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long t = __shfl_up_sync(~0u, x, d);
        if (lane >= d) x = op(t, x);
    }
    if (lane == 31) sh[w] = x;
    __syncthreads();
    if (w == 0) {
        unsigned long long y = lane < kW ? sh[lane] : 0ull;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long t = __shfl_up_sync(~0u, y, d);
            if (lane >= d && lane < kW) y = op(t, y);
        }
        if (lane < kW) sh[lane] = y;
    }
    __syncthreads();
    unsigned long long before = __shfl_up_sync(~0u, x, 1);
    const unsigned long long wpre = w ? op(init, sh[w - 1]) : init;
    before = lane ? op(wpre, before) : wpre;
    *total = op(init, sh[kW - 1]);
    __syncthreads();                                    // sh is reused by the next scan
    return before;
}

// the thread's 16 items (255 outside the slice: ignored like any non-binary value)
struct Items {
    unsigned char v[kPerThread];
    long long rel0;                                     // slice index of v[0]
};

__device__ __forceinline__ Items load_items(const unsigned char *base, long long h, unsigned long long n, unsigned long long tile) {
    Items it;
    const long long off = (long long)tile * kTile + threadIdx.x * kPerThread;
    it.rel0 = off - h;
    const unsigned char *p = base + off;
    if (it.rel0 >= 0 && it.rel0 + kPerThread <= (long long)n) {
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(p));
        const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < kPerThread; j++) it.v[j] = (unsigned char)(w[j >> 2] >> (8 * (j & 3)));
    } else {
#pragma unroll
        for (int j = 0; j < kPerThread; j++) {
            const long long r = it.rel0 + j;
            it.v[j] = (r >= 0 && r < (long long)n) ? __ldg(p + j) : (unsigned char)255;
        }
    }
    return it;
}

__global__ void __launch_bounds__(kTileThreads)
tile_summary(const unsigned char *__restrict__ base, long long h, unsigned long long n, TileRec *__restrict__ rec) {
    __shared__ unsigned long long sh[kTileThreads / 32 + 1];
    const Items it = load_items(base, h, n, blockIdx.x);
    int lv = -1, fv = -1;
    long long frel = -1, le = -1, lrel = -1;
#pragma unroll
    for (int j = 0; j < kPerThread; j++) {
        const int v = it.v[j];
        if (v > 1) continue;
        const long long r = it.rel0 + j;
        if (lv < 0) { fv = v; frel = r; }
        else if (v != lv) le = r;
        lv = v;
        lrel = r;
    }
    const unsigned long long kb = lv >= 0 ? (((unsigned long long)(lrel + 1)) << 1) | (unsigned)lv : 0ull;
    unsigned long long last_bin;
    const unsigned long long prev = block_excl<kTileThreads>(kb, 0ull, Max(), sh, &last_bin);
    if (fv >= 0 && prev != 0 && (int)(prev & 1) != fv && le < 0) le = frel;   // the thread's first edge is local
    unsigned long long edge;
    block_excl<kTileThreads>(le >= 0 ? (unsigned long long)(le + 1) : 0ull, 0ull, Max(), sh, &edge);
    // the first binary item: the max of its complement
    unsigned long long nfirst;
    block_excl<kTileThreads>(fv >= 0 ? ~((((unsigned long long)frel) << 1) | (unsigned)fv) : 0ull, 0ull, Max(), sh, &nfirst);
    if (threadIdx.x == 0) rec[blockIdx.x] = TileRec{last_bin, ~nfirst, edge};
}

// each tile's entry level and incoming since; the state's level and since after the slice
__global__ void __launch_bounds__(kScanThreads)
tile_scan(const TileRec *__restrict__ rec, unsigned long long ntiles, KfState *__restrict__ st,
          unsigned *__restrict__ entry_level, unsigned long long *__restrict__ entry_since) {
    __shared__ unsigned long long sh[kScanThreads / 32 + 1];
    const unsigned long long pos0 = st->pos0;
    unsigned long long lk = st->level, since = st->since;        // level key: (rel + 1) << 1 | value, carried = value
    for (unsigned long long t0 = 0; t0 < ntiles; t0 += kScanThreads) {
        const unsigned long long t = t0 + threadIdx.x;
        const TileRec r = t < ntiles ? rec[t] : TileRec{0ull, kNone, 0ull};
        unsigned long long lk_all;
        const unsigned long long lin = block_excl<kScanThreads>(r.last_bin, lk, Max(), sh, &lk_all);
        const unsigned level = (unsigned)(lin & 1);
        unsigned long long e = 0;
        if (r.local_edge) e = pos0 + r.local_edge - 1;
        else if (r.first_bin != kNone && (unsigned)(r.first_bin & 1) != level) e = pos0 + (r.first_bin >> 1);
        unsigned long long s_all;
        const unsigned long long sin = block_excl<kScanThreads>(e, since, Max(), sh, &s_all);
        if (t < ntiles) { entry_level[t] = level; entry_since[t] = sin; }
        lk = lk_all;
        since = s_all;
    }
    if (threadIdx.x == 0) { st->level = (unsigned)(lk & 1); st->since = since; }
}

__device__ __forceinline__ unsigned edge_kind(unsigned long long diff) {
    if (diff >= 63 && diff <= 83) return kShort;
    if (diff >= 131 && diff <= 161) return kLong;
    return kFlush;
}

// event = rel << 3 | kind << 1 | falling
__global__ void __launch_bounds__(kTileThreads)
tile_events(const unsigned char *__restrict__ base, long long h, unsigned long long n, const KfState *__restrict__ st,
            const unsigned *__restrict__ entry_level, const unsigned long long *__restrict__ entry_since,
            unsigned long long *__restrict__ events, unsigned *__restrict__ counts) {
    __shared__ unsigned long long sh[kTileThreads / 32 + 1];
    const unsigned long long tile = blockIdx.x, pos0 = st->pos0;
    const Items it = load_items(base, h, n, tile);
    int lv = -1;
    long long lrel = -1;
#pragma unroll
    for (int j = 0; j < kPerThread; j++)
        if (it.v[j] <= 1) { lv = it.v[j]; lrel = it.rel0 + j; }
    const unsigned long long kb = lv >= 0 ? (((unsigned long long)(lrel + 1)) << 1) | (unsigned)lv : 0ull;
    unsigned long long tot;
    const unsigned long long lin = block_excl<kTileThreads>(kb, entry_level[tile], Max(), sh, &tot);
    // the thread's edges from its entry level: the last one's position
    unsigned level = (unsigned)(lin & 1);
    unsigned long long last_edge = 0;
#pragma unroll
    for (int j = 0; j < kPerThread; j++) {
        const unsigned v = it.v[j];
        if (v <= 1 && v != level) { level = v; last_edge = pos0 + (unsigned long long)(it.rel0 + j); }
    }
    unsigned long long since = block_excl<kTileThreads>(last_edge, entry_since[tile], Max(), sh, &tot);
    // classes; the key of the thread's last edge: (rel + 1) << 1 | (short or long)
    level = (unsigned)(lin & 1);
    unsigned edges = 0;                                 // bit j: item j is an edge, of class (kinds >> 2 j) & 3
    unsigned long long ck = 0, kinds = 0;
#pragma unroll
    for (int j = 0; j < kPerThread; j++) {
        const unsigned v = it.v[j];
        if (v <= 1 && v != level) {
            level = v;
            const unsigned long long pos = pos0 + (unsigned long long)(it.rel0 + j);
            const unsigned k = edge_kind(pos - since);
            since = pos;
            edges |= 1u << j;
            kinds |= (unsigned long long)k << (2 * j);
            ck = (((unsigned long long)(it.rel0 + j + 1)) << 1) | (k != kFlush ? 1u : 0u);
        }
    }
    // the edge before the thread's first one: tile entry counts as short / long, so the tile's first flush is kept
    const unsigned long long pk = block_excl<kTileThreads>(ck, 1ull, Max(), sh, &tot);
    unsigned keep = 0, prev_ab = (unsigned)(pk & 1);
#pragma unroll
    for (int j = 0; j < kPerThread; j++) {
        if (!((edges >> j) & 1u)) continue;
        const unsigned k = (unsigned)(kinds >> (2 * j)) & 3u;
        if (k != kFlush || prev_ab) keep |= 1u << j;
        prev_ab = k != kFlush;
    }
    unsigned long long cnt_all;
    unsigned long long slot = block_excl<kTileThreads>((unsigned long long)__popc(keep), 0ull, Sum(), sh, &cnt_all);
    unsigned long long *ev = events + tile * kEvCap;
#pragma unroll
    for (int j = 0; j < kPerThread; j++) {
        if (!((keep >> j) & 1u)) continue;
        const unsigned k = (unsigned)(kinds >> (2 * j)) & 3u;
        ev[slot++] = ((unsigned long long)(it.rel0 + j) << 3) | (k << 1) | (it.v[j] == 0 ? 1u : 0u);
    }
    if (threadIdx.x == 0) counts[tile] = (unsigned)cnt_all;
}

// output-flag functions on {0,1}, bit x = f(x): identity 0b10, toggle 0b01, constant 0 0b00
__device__ __forceinline__ unsigned compose(unsigned later, unsigned earlier) {
    return ((later >> (earlier & 1)) & 1u) | (((later >> ((earlier >> 1) & 1)) & 1u) << 1);
}

__device__ __forceinline__ int label_of(unsigned last8) {
    return last8 == 0xD5u ? B2S_KEYFOB_CLOSE : last8 == 0xE3u ? B2S_KEYFOB_OPEN : last8 == 0xB9u ? B2S_KEYFOB_TRUNK
                                                                                                 : B2S_KEYFOB_NONE;
}

__global__ void __launch_bounds__(32)
walk_kernel(const unsigned long long *__restrict__ events, const unsigned *__restrict__ counts,
            unsigned long long ntiles, unsigned long long n, KfState *__restrict__ st, Code *__restrict__ codes) {
    __shared__ unsigned cap[8];
    const unsigned lane = threadIdx.x, lt = (1u << lane) - 1u;
    const unsigned long long pos0 = st->pos0;
    unsigned long long str_len = st->str_len, pre = st->pre, n_codes = st->n_codes;
    unsigned flag = st->flag, last32 = st->last32;
    if (lane < 8) cap[lane] = st->cap[lane];
    __syncwarp();
    unsigned long long t = 0;
    unsigned i = 0;
    while (t < ntiles) {
        const unsigned long long tt = t + lane;
        const unsigned full = tt < ntiles ? counts[tt] : 0u;
        const unsigned c = lane == 0 ? full - i : full;
        unsigned p = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned y = __shfl_up_sync(~0u, p, d);
            if (lane >= (unsigned)d) p += y;
        }
        const unsigned total = __shfl_sync(~0u, p, 31);
        if (total == 0) { t += 32; i = 0; continue; }
        const unsigned take = min(total, 32u);
        // lane L < take reads the L-th event from the cursor: its tile is the last non-empty one starting at or before L
        const unsigned start = p - c;
        const unsigned starts = __reduce_or_sync(~0u, (c > 0 && start < 32) ? 1u << start : 0u);
        const unsigned ne = __ballot_sync(~0u, c > 0);
        const bool valid = lane < take;
        const unsigned r = __popc(starts & (lt | (1u << lane)));
        unsigned tl = valid ? __fns(ne, 0, (int)r) : 0u;
        if (tl > 31) tl = 0;
        const unsigned st_tl = __shfl_sync(~0u, start, tl);
        const unsigned idx = lane - st_tl + (tl == 0 ? i : 0u);
        const unsigned long long ev = valid ? events[(t + tl) * kEvCap + idx] : 0ull;
        // the cursor after this step
        const unsigned tl_last = __shfl_sync(~0u, tl, take - 1), idx_last = __shfl_sync(~0u, idx, take - 1);
        const unsigned full_last = __shfl_sync(~0u, full, tl_last);
        t += tl_last;
        i = idx_last + 1;
        if (i >= full_last) { t++; i = 0; }

        const unsigned kind = valid ? (unsigned)(ev >> 1) & 3u : (unsigned)kFlush + 1u;
        const unsigned f = kind == kShort ? 0b01u : kind == kLong ? 0b00u : 0b10u;
        unsigned incl = f;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned y = __shfl_up_sync(~0u, incl, d);
            if (lane >= (unsigned)d) incl = compose(incl, y);
        }
        unsigned excl = __shfl_up_sync(~0u, incl, 1);
        if (lane == 0) excl = 0b10u;
        const unsigned before = (excl >> flag) & 1u;
        const bool append = kind == kLong || (kind == kShort && before);
        const unsigned bit = (unsigned)(ev & 1u);              // falling edge: "1"
        const unsigned am = __ballot_sync(~0u, append);
        unsigned cm = __ballot_sync(~0u, kind == kFlush);
        flag = (__shfl_sync(~0u, incl, 31) >> flag) & 1u;
        // with no bit appended in this step only the first flush can act, and only on a non-empty string
        if (!am) cm = str_len ? cm & (0u - cm) : 0u;

        unsigned lo = 0;
        while (true) {
            const unsigned rest = lo < 32 ? cm & (~0u << lo) : 0u;
            const unsigned cpos = rest ? (unsigned)__ffs(rest) - 1u : 32u;
            const unsigned gm = am & (lo < 32 ? ~0u << lo : 0u) & (cpos < 32 ? (1u << cpos) - 1u : ~0u);
            if (gm) {                                   // the bits these lanes append, oldest first
                const unsigned k = __popc(gm);
                const bool mine = (gm >> lane) & 1u;
                const unsigned j = __popc(gm & lt);
                const unsigned nb = __reduce_or_sync(~0u, mine && bit ? 1u << (k - 1 - j) : 0u);
                const unsigned long long w = ((unsigned long long)last32 << k) | nb;
                // a match ends at the bit of rank q (q < k) if all 8 of its bits are in the string
                const bool m = lane < k && str_len + lane + 1 >= 8 &&
                               (unsigned)((w >> (k - 1 - lane)) & 0xFFu) == kPreamble;
                const unsigned mm = __ballot_sync(~0u, m);
                if (pre == kNone && mm) {
                    pre = str_len + (unsigned)__ffs(mm) - 8;   // ffs - 1 + 1 - 8
                    if (lane == 0) cap[0] = kPreamble;
                    __syncwarp();
                }
                if (pre != kNone && mine && bit) {
                    const unsigned long long off = str_len + j - pre;
                    if (off >= 8 && off < 256) {
                        const unsigned b = (unsigned)off >> 3;
                        atomicOr(&cap[b >> 2], 1u << ((b & 3u) * 8u + 7u - ((unsigned)off & 7u)));
                    }
                }
                __syncwarp();
                str_len += k;
                last32 = (unsigned)w;
            }
            if (cpos >= 32) break;
            // print(): a string with a preamble is reported from it on (it then has >= 8 bits)
            if (pre != kNone) {
                const unsigned long long rel = __shfl_sync(~0u, ev, cpos) >> 3;
                Code *cd = codes + n_codes;
                if (lane < 8) reinterpret_cast<unsigned *>(cd->bits)[lane] = cap[lane];
                if (lane == 0) {
                    const unsigned long long nb = str_len - pre;
                    cd->index = pos0 + rel;
                    cd->n_bits = nb > 0xFFFFFFFFull ? 0xFFFFFFFFu : (unsigned)nb;
                    cd->label = label_of(last32 & 0xFFu);
                }
                __syncwarp();
                if (lane < 8) cap[lane] = 0u;
                n_codes++;
            }
            __syncwarp();
            str_len = 0;
            pre = kNone;
            last32 = 0;
            lo = cpos + 1;
        }
    }
    if (lane < 8) st->cap[lane] = cap[lane];
    if (lane == 0) {
        st->pos0 = pos0 + n;
        st->n_codes = n_codes;
        st->str_len = str_len;
        st->pre = pre;
        st->flag = flag;
        st->last32 = last32;
    }
}

}  // namespace

struct b2s_keyfob {
    b2s_ctx *ctx = nullptr;
    Buf<KfState> st;
    Buf<Code> codes;
    Buf<TileRec> rec;
    Buf<unsigned> level, counts;
    Buf<unsigned long long> since, events;
    size_t cd_bound = 0, cd_rd = 0;    // upper bound of the list's length, entries already drained
    ListCounts<1> count;               // n_codes as the last exec left it
};

extern "C" {

int32_t b2s_keyfob_create(b2s_ctx *ctx, b2s_keyfob **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_keyfob_create: NULL argument");
    *out = nullptr;
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_keyfob> p(new b2s_keyfob());
    p->ctx = ctx;
    B2S_TRY(p->st.alloc(ctx, 1, "b2s_keyfob_create: state"));
    B2S_TRY(p->count.init(ctx, "b2s_keyfob_create: list count"));
    B2S_TRY(b2s_keyfob_reset(p.get()));
    *out = p.release();
    return B2S_OK;
}

void b2s_keyfob_destroy(b2s_keyfob *p) { PlanDeleter<b2s_keyfob>()(p); }

// State::Down(0), output = false, an empty string, no codes (decoder.rs:26-34)
int32_t b2s_keyfob_reset(b2s_keyfob *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "keyfob is NULL");
    DeviceGuard g(p->ctx->device);
    B2S_TRY(b2s_memset(p->ctx, p->st.get(), 0, sizeof(KfState)));
    B2S_TRY(b2s_memset(p->ctx, &p->st.get()->pre, 0xFF, sizeof(unsigned long long)));
    p->cd_bound = p->cd_rd = 0;
    p->count.pending = false;
    return B2S_OK;
}

int32_t b2s_keyfob_exec(b2s_keyfob *p, const uint8_t *d_in, size_t n_in, size_t *consumed) {
    if (!p || !consumed) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_keyfob_exec: NULL argument");
    *consumed = 0;
    if (n_in == 0) return B2S_OK;
    b2s_ctx *ctx = p->ctx;
    if (!d_in) return b2s_fail(ctx, B2S_EINVAL, "b2s_keyfob_exec: NULL slice");
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_keyfob_exec");
    const long long h = (long long)((uintptr_t)d_in & 15);
    const unsigned char *base = d_in - h;
    const size_t ntiles = ceil_div(n_in + (size_t)h, kTile);
    if (ntiles > 0x7FFFFFFFull) return b2s_fail(ctx, B2S_EINVAL, "b2s_keyfob_exec: %zu items in one exec", n_in);
    // every appended bit is >= 63 items after the previous edge and a code needs >= 8 bits
    const size_t bound_new = n_in / (8 * 63) + 2;
    B2S_TRY(p->count.refresh(ctx, p->codes.size() < p->cd_bound + bound_new, {&p->cd_bound}));
    B2S_TRY(list_grow(ctx, p->codes, p->cd_bound + bound_new, p->cd_bound, "b2s_keyfob_exec: code list"));
    B2S_TRY(p->rec.reserve(ctx, ntiles, "b2s_keyfob_exec: tile records"));
    B2S_TRY(p->level.reserve(ctx, ntiles, "b2s_keyfob_exec: tile levels"));
    B2S_TRY(p->since.reserve(ctx, ntiles, "b2s_keyfob_exec: tile since"));
    B2S_TRY(p->counts.reserve(ctx, ntiles, "b2s_keyfob_exec: tile event counts"));
    B2S_TRY(p->events.reserve(ctx, ntiles * kEvCap, "b2s_keyfob_exec: events"));
    KfState *st = p->st.get();
    tile_summary<<<(unsigned)ntiles, kTileThreads, 0, ctx->stream>>>(base, h, n_in, p->rec.get());
    B2S_CHECK_LAUNCH(ctx);
    tile_scan<<<1, kScanThreads, 0, ctx->stream>>>(p->rec.get(), ntiles, st, p->level.get(), p->since.get());
    B2S_CHECK_LAUNCH(ctx);
    tile_events<<<(unsigned)ntiles, kTileThreads, 0, ctx->stream>>>(base, h, n_in, st, p->level.get(), p->since.get(),
                                                                      p->events.get(), p->counts.get());
    B2S_CHECK_LAUNCH(ctx);
    walk_kernel<<<1, 32, 0, ctx->stream>>>(p->events.get(), p->counts.get(), ntiles, n_in, st, p->codes.get());
    B2S_CHECK_LAUNCH(ctx);
    B2S_TRY(p->count.record(ctx, &st->n_codes));
    p->cd_bound += bound_new;
    *consumed = n_in;
    return B2S_OK;
}

int32_t b2s_keyfob_drain_codes(b2s_keyfob *p, b2s_keyfob_code *host, size_t cap, size_t *n) {
    if (!p || !n || (cap && !host)) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_keyfob_drain_codes: NULL argument");
    return list_drain(p->ctx, p->codes, &p->st.get()->n_codes, p->count, p->cd_rd, p->cd_bound, host, cap, n,
                      [](const Code &) { return true; });
}

}  // extern "C"
