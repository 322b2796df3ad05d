// lora.cu -- the LoRa transmitter (examples/lora/src/{encoder,modulator,transmitter}.rs and the chirp helpers of
// utils.rs:917-963) as a device source (DESIGN §4.19).
//
// Encoder (encoder.rs:33-284): one warp per frame.  The warp stages the payload in shared memory, lane 0 runs the
// CRC-16, the lanes build the Hamming codewords of every nibble (whitened payload, explicit header, CRC), and each lane
// then forms whole symbols: symbol i of an interleaver block takes bit i of the block's codewords on the diagonal, then
// the LDRO parity bit, the gray demap and the +1.
//
// Modulator (modulator.rs:46-152, samples_from_phase_diff): every sample of a frame is exp(i S[k]) with
// S[k] = S[k-1] + p[k] in f32 from +0, in order.  The increments p are closed-form; the running sum is not: no scan
// reassociation gives the reference's bits.  So each frame's sum is one dependent chain, and parallelism comes from
// frames: a CTA takes up to 32 frames (jobs), lane l of warp 0 walks job l's chain over shared-memory chunks, while the
// other warps write the next chunk's increments and turn the previous chunk's phases into samples (f64 sincos rounded
// once to f32) with coalesced stores.  A frame cut by the end of an exec keeps its S in its device record, and the next
// exec resumes from there: execs never synchronise.
//
// Numerics: __ddiv_rn / __dsub_rn / __double2float_rn / __fdiv_rn / __fadd_rn / __fmul_rn in the reference's order, no
// contraction, so increments and phase sums are the reference's bits.
#include <algorithm>
#include <cmath>
#include <cstdint>

#include "common.cuh"
#include "tx_common.cuh"

namespace {

// ---- configuration ----------------------------------------------------------------------------------------------
struct LoraCfg {
    int sf, cr, has_crc, ldro, implicit;
};

// the first interleaver block: header (or, implicit, the first payload nibbles) at CR 4/8; SF < 7 never uses LDRO
// there (encoder.rs:195-215); later blocks use `sf - 2` nibbles only with LDRO
__host__ __device__ inline int sf_app0(const LoraCfg &c) { return c.sf >= 7 ? c.sf - 2 : c.sf; }
__host__ __device__ inline int sf_app1(const LoraCfg &c) { return c.ldro ? c.sf - 2 : c.sf; }

int32_t check_cfg(b2s_ctx *ctx, const LoraCfg &c, const char *what) {
    if (c.sf < 5 || c.sf > 12) return b2s_fail(ctx, B2S_EINVAL, "%s: spreading factor %d is not 5..12", what, c.sf);
    if (c.cr < 1 || c.cr > 4) return b2s_fail(ctx, B2S_EINVAL, "%s: code rate %d is not 1..4", what, c.cr);
    return B2S_OK;
}

// nibbles before interleaving: header, whitened payload, CRC (encoder.rs:33-53)
size_t nibble_count(const LoraCfg &c, size_t len) { return (c.implicit ? 0 : 5) + 2 * len + (c.has_crc ? 4 : 0); }

// interleave() always emits at least one block, even for an empty frame (encoder.rs:193-265)
size_t symbol_count(const LoraCfg &c, size_t len) {
    const size_t m = nibble_count(c, len), a0 = (size_t)sf_app0(c), a1 = (size_t)sf_app1(c);
    const size_t blocks = m <= a0 ? 1 : 1 + ceil_div(m - a0, a1);
    return 8 + (blocks - 1) * (4 + (size_t)c.cr);
}

int32_t check_payload(b2s_ctx *ctx, const LoraCfg &c, size_t len, const char *what) {
    if (len > 255) return b2s_fail(ctx, B2S_EINVAL, "%s: a payload of %zu bytes (at most 255)", what, len);
    if (c.has_crc && len < 2)
        return b2s_fail(ctx, B2S_EINVAL, "%s: a payload of %zu bytes with CRC (at least 2)", what, len);
    return B2S_OK;
}

// ---- encoder ----------------------------------------------------------------------------------------------------
constexpr int kEncWarps = 4;
constexpr int kMaxNibbles = 5 + 2 * 255 + 4;

struct EncFrame {
    unsigned long long byte_off, sym_abs;   // payload bytes; first symbol (ring index before the mask)
    unsigned len;
};

// WHITENING_SEQ (utils.rs:40): the LFSR x^8 + x^6 + x^5 + x^4 + 1 from 0xFF, shifting left, the new bit the parity of
// bits 7, 5, 4 and 3
struct Whitening {
    unsigned char seq[255];
    constexpr Whitening() : seq() {
        unsigned s = 0xFF;
        for (int i = 0; i < 255; ++i) {
            seq[i] = (unsigned char)s;
            unsigned t = s & 0xB8u, par = 0;
            for (; t; t &= t - 1) par ^= 1u;
            s = ((s << 1) | par) & 0xFFu;
        }
    }
};
__constant__ Whitening kWhitening = Whitening();

// crc16 (encoder.rs:105-117), one byte
__device__ unsigned crc16_step(unsigned crc, unsigned byte) {
    for (int i = 0; i < 8; ++i) {
        crc = (((crc & 0x8000u) >> 8) ^ (byte & 0x80u)) ? ((crc << 1) ^ 0x1021u) : (crc << 1);
        crc &= 0xFFFFu;
        byte = (byte << 1) & 0xFFFFu;
    }
    return crc;
}

// hamming_encode (encoder.rs:134-182) of one nibble at rate cr_app; b0 is the nibble's LSB (data_bin[3])
__device__ unsigned hamming(unsigned nib, int cr_app) {
    const unsigned b0 = nib & 1u, b1 = (nib >> 1) & 1u, b2 = (nib >> 2) & 1u, b3 = (nib >> 3) & 1u;
    if (cr_app == 1) return b0 << 4 | b1 << 3 | b2 << 2 | b3 << 1 | (b0 ^ b1 ^ b2 ^ b3);
    const unsigned p0 = b0 ^ b1 ^ b2, p1 = b1 ^ b2 ^ b3, p2 = b0 ^ b1 ^ b3, p3 = b0 ^ b2 ^ b3;
    return (b0 << 7 | b1 << 6 | b2 << 5 | b3 << 4 | p0 << 3 | p1 << 2 | p2 << 1 | p3) >> (4 - cr_app);
}

__global__ void __launch_bounds__(kEncWarps * 32) lora_encode_kernel(const unsigned char *bytes,
                                                                      const EncFrame *frames, unsigned n_frames,
                                                                      LoraCfg c, unsigned short *sym,
                                                                      unsigned long long sym_mask) {
    __shared__ unsigned char s_pay[kEncWarps][256];
    __shared__ unsigned char s_cw[kEncWarps][kMaxNibbles + 1];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned f = blockIdx.x * kEncWarps + w;
    if (f >= n_frames) return;
    const EncFrame fr = frames[f];
    const unsigned len = fr.len;
    unsigned char *pay = s_pay[w], *cw = s_cw[w];
    for (unsigned i = lane; i < len; i += 32) pay[i] = bytes[fr.byte_off + i];
    __syncwarp();
    unsigned crc = 0;
    if (c.has_crc && lane == 0) {            // encoder.rs:119-132: all but the last two bytes, then XOR them
        for (unsigned i = 0; i + 2 < len; ++i) crc = crc16_step(crc, pay[i]);
        crc ^= pay[len - 1] ^ ((unsigned)pay[len - 2] << 8);
    }
    crc = __shfl_sync(~0u, crc, 0);
    // header (encoder.rs:64-103)
    const unsigned h0 = len >> 4, h1 = len & 0xFu, h2 = ((unsigned)c.cr << 1) | (unsigned)c.has_crc;
    const unsigned c4 = ((h0 >> 3) ^ (h0 >> 2) ^ (h0 >> 1) ^ h0) & 1u;
    const unsigned c3 = ((h0 >> 3) ^ (h1 >> 3) ^ (h1 >> 2) ^ (h1 >> 1) ^ h2) & 1u;
    const unsigned c2 = ((h0 >> 2) ^ (h1 >> 3) ^ h1 ^ (h2 >> 3) ^ (h2 >> 1)) & 1u;
    const unsigned c1 = ((h0 >> 1) ^ (h1 >> 2) ^ h1 ^ (h2 >> 2) ^ (h2 >> 1) ^ h2) & 1u;
    const unsigned c0 = (h0 ^ (h1 >> 1) ^ (h2 >> 3) ^ (h2 >> 2) ^ (h2 >> 1) ^ h2) & 1u;
    const unsigned hdr = c.implicit ? 0u : 5u;
    const unsigned m = hdr + 2 * len + (c.has_crc ? 4u : 0u);
    const int a0 = sf_app0(c), a1 = sf_app1(c);
    for (unsigned k = lane; k < m; k += 32) {
        unsigned nib;
        if (k < hdr) nib = k == 0 ? h0 : k == 1 ? h1 : k == 2 ? h2 : k == 3 ? c4 : (c3 << 3 | c2 << 2 | c1 << 1 | c0);
        else if (k < hdr + 2 * len) {        // whitening (encoder.rs:55-62)
            const unsigned i = k - hdr, b = pay[i >> 1] ^ kWhitening.seq[i >> 1];
            nib = (i & 1u) ? b >> 4 : b & 0xFu;
        } else nib = (crc >> (4 * (k - hdr - 2 * len))) & 0xFu;
        cw[k] = (unsigned char)hamming(nib, (int)k < a0 ? 4 : c.cr);
    }
    __syncwarp();
    // interleave (encoder.rs:184-268) + gray_demap (:270-284), one symbol per lane
    const unsigned n_sym = m <= (unsigned)a0 ? 8u : 8u + ((m - a0 + a1 - 1) / a1) * (4u + c.cr);
    const unsigned nmask = (1u << c.sf) - 1u;
    for (unsigned s = lane; s < n_sym; s += 32) {
        int cw_len, sf_app, row;
        bool use_ldro;
        unsigned base;
        if (s < 8) {
            cw_len = 8; sf_app = a0; use_ldro = c.sf >= 7; row = (int)s; base = 0;
        } else {
            const unsigned b = (s - 8) / (4u + c.cr);
            cw_len = 4 + c.cr; sf_app = a1; use_ldro = c.ldro != 0; row = (int)(s - 8 - b * (4u + c.cr));
            base = (unsigned)a0 + b * (unsigned)a1;
        }
        unsigned v = 0;
        for (int j = 0; j < sf_app; ++j) {
            const int k = ((row - j - 1) % sf_app + sf_app) % sf_app;
            const unsigned word = base + k < m ? cw[base + k] : 0u;
            v |= ((word >> (cw_len - 1 - row)) & 1u) << (c.sf - 1 - j);
        }
        if (use_ldro) v |= (unsigned)(__popc(v) & 1) << (c.sf - 1 - sf_app);
        unsigned g = v;
        for (int j = 1; j < c.sf; ++j) g ^= v >> j;
        sym[(fr.sym_abs + s) & sym_mask] = (unsigned short)((g + 1u) & nmask);
    }
}

int32_t launch_encode(b2s_ctx *ctx, const unsigned char *bytes, const EncFrame *frames, size_t n, const LoraCfg &c,
                      unsigned short *sym, unsigned long long mask) {
    if (!n) return B2S_OK;
    lora_encode_kernel<<<(unsigned)ceil_div(n, kEncWarps), kEncWarps * 32, 0, ctx->stream>>>(bytes, frames,
                                                                                           (unsigned)n, c, sym, mask);
    B2S_CHECK_LAUNCH(ctx);
    return B2S_OK;
}

// ---- modulator --------------------------------------------------------------------------------------------------
constexpr int kJobs = 32;              // frames per CTA: one lane of warp 0 each
constexpr int kCh = 128;               // samples of each job per chunk
constexpr int kRow = kJobs + 1;        // shared row of one chunk position: the 32 jobs, padded against bank conflicts
constexpr int kStages = 3;             // being filled with increments / being summed / being turned into samples
constexpr int kModThreads = 512;
constexpr size_t kModSmem = (size_t)kStages * kCh * kRow * sizeof(float);

struct TxFrame {                       // device record of one queued frame
    unsigned long long start, sym_abs; // stream index of its first sample; its first symbol
    unsigned n_sym;
    unsigned short sync0, sync1;       // the sync word it was started with
    float S;                           // the phase sum after the last sample produced, while the frame is cut
    unsigned pad_;
};

struct ModParams {
    const float *A;                    // A[t] = (float)((double)t / N - 0.5), t < N
    const unsigned short *sym;
    unsigned long long sym_mask;
    TxFrame *frames;
    unsigned long long frame_mask, f_lo;
    unsigned n_jobs, jpc;
    unsigned long long pos, cnt;       // this exec's stream samples [pos, pos + cnt)
    float2 *out;
    unsigned N, Q, pad, P, extra, base_len, sf;
    float k_up, k_down;                // (polarity * (1 / OS)) * (2 PI)
    unsigned short sync0, sync1;       // the sync word for frames that start in this exec
};

struct Job {
    unsigned long long out_off, sym_abs, frame;
    unsigned j0, cnt, n_sym;
    unsigned short s0, s1;
    bool resume, cut;
};

// build_upchirp_phase_coherent (utils.rs:917-951) at sample j of the frame, laid out as modulate() does
__device__ __forceinline__ float increment(const ModParams &m, const Job &jb, unsigned j) {
    if (j < m.pad) return 0.0f;
    j -= m.pad;
    unsigned t;
    int id = 0;
    bool up = true;
    const unsigned pre = (m.P + 4) * m.N;
    if (j < pre) {                     // preamble upchirps, two sync upchirps, two downchirps
        const unsigned c = j / m.N;
        t = j - c * m.N;
        if (c == m.P) id = jb.s0;
        else if (c == m.P + 1) id = jb.s1;
        else if (c > m.P + 1) up = false;
    } else if ((j -= pre) < m.Q) {     // the quarter downchirp
        t = j;
        up = false;
    } else if ((j -= m.Q) < m.extra) { // SF < 7: two more upchirps
        t = j % m.N;
    } else {                           // data upchirps with offset_id, then the tail pad
        j -= m.extra;
        const unsigned c = j / m.N;
        if (c >= jb.n_sym) return 0.0f;
        t = j - c * m.N;
        id = (int)m.sym[(jb.sym_abs + c) & m.sym_mask] - 1;
    }
    float p = __fadd_rn(m.A[t], __fdiv_rn((float)id, (float)(1u << m.sf)));
    if (p > 0.5f) p = __fsub_rn(p, 1.0f);
    else if (p < -0.5f) p = __fadd_rn(p, 1.0f);
    return __fmul_rn(p, up ? m.k_up : m.k_down);
}

__global__ void lora_table_kernel(float *A, unsigned N) {
    for (unsigned t = blockIdx.x * blockDim.x + threadIdx.x; t < N; t += gridDim.x * blockDim.x)
        A[t] = __double2float_rn(__dsub_rn(__ddiv_rn((double)t, (double)N), 0.5));
}

__global__ void __launch_bounds__(kModThreads, 2) lora_mod_kernel(ModParams m) {
    extern __shared__ float s_buf[];
    __shared__ Job s_job[kJobs];
    __shared__ unsigned s_chunks;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned first = blockIdx.x * m.jpc;
    const unsigned nj = min(m.jpc, m.n_jobs - first);
    if (threadIdx.x == 0) s_chunks = 0;
    __syncthreads();
    float S = 0.0f;
    if (warp == 0 && (unsigned)lane < nj) {
        const unsigned long long f = m.f_lo + first + lane;
        TxFrame *rec = m.frames + (f & m.frame_mask);
        const unsigned long long start = rec->start, len = m.base_len + (unsigned long long)rec->n_sym * m.N;
        const unsigned long long a = max(m.pos, start), b = min(m.pos + m.cnt, start + len);
        Job jb;
        jb.out_off = a - m.pos;
        jb.sym_abs = rec->sym_abs;
        jb.frame = f;
        jb.j0 = (unsigned)(a - start);
        jb.cnt = (unsigned)(b - a);
        jb.n_sym = rec->n_sym;
        jb.resume = jb.j0 > 0;
        jb.cut = b < start + len;
        if (jb.resume) {
            jb.s0 = rec->sync0; jb.s1 = rec->sync1;
            S = rec->S;
        } else {                       // the sync word is latched when a frame's first sample is produced
            jb.s0 = rec->sync0 = m.sync0; jb.s1 = rec->sync1 = m.sync1;
        }
        s_job[lane] = jb;
        atomicMax(&s_chunks, (jb.cnt + kCh - 1) / kCh);
    }
    __syncthreads();
    const unsigned nch = s_chunks;
    const int h = threadIdx.x - 32, H = kModThreads - 32;
    for (unsigned s = 0; s < nch + 2; ++s) {
        if (warp == 0) {
            if (s >= 1 && s <= nch) {  // one dependent f32 add per sample, in order (samples_from_phase_diff)
                float *buf = s_buf + (size_t)((s - 1) % kStages) * kCh * kRow + lane;
#pragma unroll 16
                for (int k = 0; k < kCh; ++k) {
                    S = __fadd_rn(S, buf[k * kRow]);
                    buf[k * kRow] = S;
                }
            }
        } else {
            if (s < nch) {             // increments of chunk s; past a job's end they are 0 and leave S unchanged
                float *buf = s_buf + (size_t)(s % kStages) * kCh * kRow;
                for (unsigned idx = h; idx < nj * kCh; idx += H) {
                    const unsigned l = idx / kCh, k = idx % kCh, r = s * kCh + k;
                    const Job &jb = s_job[l];
                    buf[k * kRow + l] = r < jb.cnt ? increment(m, jb, jb.j0 + r) : 0.0f;
                }
            }
            if (s >= 2) {              // samples of chunk s - 2: (1 + 0i) * from_polar(1, S)
                const unsigned c = s - 2;
                const float *buf = s_buf + (size_t)(c % kStages) * kCh * kRow;
                for (unsigned idx = h; idx < nj * kCh; idx += H) {
                    const unsigned l = idx / kCh, k = idx % kCh, r = c * kCh + k;
                    const Job &jb = s_job[l];
                    if (r >= jb.cnt) continue;
                    double sd, cd;
                    sincos((double)buf[k * kRow + l], &sd, &cd);
                    const float co = __double2float_rn(cd), si = __double2float_rn(sd);
                    const float re = __fsub_rn(__fmul_rn(1.0f, co), __fmul_rn(0.0f, si));
                    const float im = __fadd_rn(__fmul_rn(1.0f, si), __fmul_rn(0.0f, co));
                    m.out[jb.out_off + r] = make_float2(re, im);
                }
            }
        }
        __syncthreads();
    }
    if (warp == 0 && (unsigned)lane < nj && s_job[lane].cut) m.frames[s_job[lane].frame & m.frame_mask].S = S;
}

}  // namespace

struct b2s_lora_tx {
    b2s_ctx *ctx = nullptr;
    LoraCfg cfg{};
    unsigned os = 1, N = 0, Q = 0, P = 0, pad = 0, extra = 0, base_len = 0;
    float k_up = 0.f, k_down = 0.f;
    unsigned short sync_create[2] = {0, 0}, sync[2] = {0, 0};
    Buf<float> A;
    DevRing<unsigned short> sym;
    DevRing<TxFrame> frames;
    Buf<unsigned char> bytes;          // the payloads of the last push
    Buf<EncFrame> enc;
    TxQueue<b2s_lora_burst> q;
};

namespace {
int32_t check_sync(b2s_ctx *ctx, int sf, uint32_t s0, uint32_t s1, const char *what) {
    // SynchWord::verify (utils.rs:465-489)
    if (s0 >= (1u << sf) || s1 >= (1u << sf))
        return b2s_fail(ctx, B2S_EINVAL, "%s: sync symbols [%u, %u] do not fit SF%d (below %u)", what, s0, s1, sf,
                        1u << sf);
    return B2S_OK;
}
}  // namespace

extern "C" {

int32_t b2s_lora_symbol_count(int32_t sf, int32_t code_rate, int32_t has_crc, int32_t ldro_enabled,
                              int32_t implicit_header, size_t payload_len, size_t *n_symbols) {
    if (!n_symbols) return b2s_fail(nullptr, B2S_EINVAL, "b2s_lora_symbol_count: NULL argument");
    const LoraCfg c{sf, code_rate, has_crc != 0, ldro_enabled != 0, implicit_header != 0};
    B2S_TRY(check_cfg(nullptr, c, "b2s_lora_symbol_count"));
    B2S_TRY(check_payload(nullptr, c, payload_len, "b2s_lora_symbol_count"));
    *n_symbols = symbol_count(c, payload_len);
    return B2S_OK;
}

int32_t b2s_lora_encode(b2s_ctx *ctx, int32_t sf, int32_t code_rate, int32_t has_crc, int32_t ldro_enabled,
                        int32_t implicit_header, const uint8_t *d_payloads, const size_t *lengths, size_t n_frames,
                        uint16_t *d_symbols, size_t symbols_cap, size_t *n_symbols) {
    if (!ctx || !n_symbols || (n_frames && !lengths)) return b2s_fail(ctx, B2S_EINVAL, "b2s_lora_encode: NULL argument");
    *n_symbols = 0;
    const LoraCfg c{sf, code_rate, has_crc != 0, ldro_enabled != 0, implicit_header != 0};
    B2S_TRY(check_cfg(ctx, c, "b2s_lora_encode"));
    std::vector<EncFrame> fr(n_frames);
    size_t nb = 0, ns = 0;
    for (size_t i = 0; i < n_frames; ++i) {
        B2S_TRY(check_payload(ctx, c, lengths[i], "b2s_lora_encode"));
        fr[i] = EncFrame{nb, ns, (unsigned)lengths[i]};
        nb += lengths[i];
        ns += symbol_count(c, lengths[i]);
    }
    if (nb && !d_payloads) return b2s_fail(ctx, B2S_EINVAL, "b2s_lora_encode: NULL payloads");
    if (ns > symbols_cap)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_lora_encode: %zu symbols do not fit %zu", ns, symbols_cap);
    if (ns && !d_symbols) return b2s_fail(ctx, B2S_EINVAL, "b2s_lora_encode: NULL symbols");
    if (!n_frames) return B2S_OK;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_lora_encode");
    // the frame table lives in stream-ordered memory: nothing waits, and it is freed after the kernel
    void *d_fr = nullptr;
    B2S_CUDA(ctx, cudaMallocAsync(&d_fr, n_frames * sizeof(EncFrame), ctx->stream));
    B2S_CUDA(ctx, cudaMemcpyAsync(d_fr, fr.data(), n_frames * sizeof(EncFrame), cudaMemcpyHostToDevice, ctx->stream));
    const int32_t rc = launch_encode(ctx, d_payloads, (const EncFrame *)d_fr, n_frames, c, d_symbols, ~0ull);
    B2S_CUDA(ctx, cudaFreeAsync(d_fr, ctx->stream));
    B2S_TRY(rc);
    *n_symbols = ns;
    return B2S_OK;
}

int32_t b2s_lora_tx_create(b2s_ctx *ctx, int32_t sf, int32_t code_rate, int32_t has_crc, int32_t ldro_enabled,
                           int32_t implicit_header, size_t oversampling, const uint32_t sync_symbols[2],
                           size_t preamble_len, size_t pad, b2s_lora_tx **out) {
    if (!ctx || !out || !sync_symbols) return b2s_fail(ctx, B2S_EINVAL, "b2s_lora_tx_create: NULL argument");
    *out = nullptr;
    const LoraCfg c{sf, code_rate, has_crc != 0, ldro_enabled != 0, implicit_header != 0};
    B2S_TRY(check_cfg(ctx, c, "b2s_lora_tx_create"));
    B2S_TRY(check_sync(ctx, sf, sync_symbols[0], sync_symbols[1], "b2s_lora_tx_create"));
    if (oversampling == 0 || oversampling > (1u << 20) || ((size_t)1 << sf) * oversampling > (1u << 20))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_lora_tx_create: 2^%d * oversampling %zu is 0 or above 2^20", sf,
                        oversampling);
    const unsigned long long N = ((unsigned long long)1 << sf) * oversampling;
    const unsigned long long extra = sf < 7 ? 2 * N : 0, Q = N / 4 - oversampling;
    // a frame's samples are indexed in 32 bits: the longest one (255 bytes with CRC) must fit
    const LoraCfg worst{sf, code_rate, 1, ldro_enabled != 0, implicit_header != 0};
    const unsigned long long base = (preamble_len + 4) * N + Q + extra;
    if (preamble_len > (1u << 20) || pad > 0xFFFFFFFFull ||
        2 * (unsigned long long)pad + base + symbol_count(worst, 255) * N > 0xFFFFFFFFull)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_lora_tx_create: a frame of preamble %zu and pad %zu exceeds 2^32 samples",
                        preamble_len, pad);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_lora_tx> p(new b2s_lora_tx());
    p->ctx = ctx;
    p->cfg = c;
    p->os = (unsigned)oversampling;
    p->N = (unsigned)N;
    p->Q = (unsigned)Q;
    p->P = (unsigned)preamble_len;
    p->pad = (unsigned)pad;
    p->extra = (unsigned)extra;
    p->base_len = (unsigned)(2 * (unsigned long long)pad + base);
    // `p *= polarity * (1.0 / os_factor as f32) * (2.0 * PI)`, left to right in f32 (utils.rs:947)
    const float two_pi = 2.0f * 3.14159265358979323846f;
    p->k_up = (1.0f * (1.0f / (float)oversampling)) * two_pi;
    p->k_down = (-1.0f * (1.0f / (float)oversampling)) * two_pi;
    p->sync_create[0] = p->sync[0] = (unsigned short)sync_symbols[0];
    p->sync_create[1] = p->sync[1] = (unsigned short)sync_symbols[1];
    B2S_TRY(p->A.alloc(ctx, N, "b2s_lora_tx_create: chirp table"));
    lora_table_kernel<<<(unsigned)ceil_div(N, 256), 256, 0, ctx->stream>>>(p->A.get(), (unsigned)N);
    B2S_CHECK_LAUNCH(ctx);
    B2S_TRY(smem_optin<lora_mod_kernel>(ctx, kModSmem));
    *out = p.release();
    return B2S_OK;
}

void b2s_lora_tx_destroy(b2s_lora_tx *p) { PlanDeleter<b2s_lora_tx>()(p); }

int32_t b2s_lora_tx_reset(b2s_lora_tx *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "lora transmitter is NULL");
    p->q.reset();
    p->sync[0] = p->sync_create[0];
    p->sync[1] = p->sync_create[1];
    return B2S_OK;
}

int32_t b2s_lora_tx_push(b2s_lora_tx *p, const uint8_t *payloads, const size_t *lengths, size_t n_frames) {
    if (!p || (n_frames && !lengths)) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_lora_tx_push: NULL argument");
    b2s_ctx *ctx = p->ctx;
    std::vector<EncFrame> enc(n_frames);
    std::vector<TxFrame> rec(n_frames);
    std::vector<TxHostFrame> hf(n_frames);
    size_t nb = 0;
    unsigned long long ns = 0, start = p->q.total;
    for (size_t i = 0; i < n_frames; ++i) {
        B2S_TRY(check_payload(ctx, p->cfg, lengths[i], "b2s_lora_tx_push"));
        const unsigned n_sym = (unsigned)symbol_count(p->cfg, lengths[i]);
        enc[i] = EncFrame{nb, p->q.s_head + ns, (unsigned)lengths[i]};
        rec[i] = TxFrame{start, p->q.s_head + ns, n_sym, 0, 0, 0.0f, 0};
        hf[i] = TxHostFrame{start, p->base_len + (unsigned long long)n_sym * p->N, p->q.s_head + ns};
        start += hf[i].len;
        nb += lengths[i];
        ns += n_sym;
    }
    if (nb && !payloads) return b2s_fail(ctx, B2S_EINVAL, "b2s_lora_tx_push: NULL payloads");
    if (!n_frames) return B2S_OK;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_lora_tx_push");
    B2S_TRY(p->frames.make_room(ctx, p->q.f_tail, p->q.f_head, n_frames, "b2s_lora_tx_push: frame records"));
    B2S_TRY(p->sym.make_room(ctx, p->q.s_tail, p->q.s_head, ns, "b2s_lora_tx_push: symbols"));
    B2S_TRY(p->bytes.reserve(ctx, std::max<size_t>(nb, 1), "b2s_lora_tx_push: payloads"));
    B2S_TRY(p->enc.reserve(ctx, n_frames, "b2s_lora_tx_push: frame table"));
    if (nb) B2S_CUDA(ctx, cudaMemcpyAsync(p->bytes.get(), payloads, nb, cudaMemcpyHostToDevice, ctx->stream));
    B2S_CUDA(ctx, cudaMemcpyAsync(p->enc.get(), enc.data(), n_frames * sizeof(EncFrame), cudaMemcpyHostToDevice,
                                  ctx->stream));
    B2S_TRY(p->frames.put(ctx, p->q.f_head, rec.data(), n_frames));
    B2S_TRY(launch_encode(ctx, p->bytes.get(), p->enc.get(), n_frames, p->cfg, p->sym.b.get(), p->sym.mask()));
    p->q.append(hf, ns);
    return B2S_OK;
}

int32_t b2s_lora_tx_set_sync_word(b2s_lora_tx *p, uint32_t sync0, uint32_t sync1) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "lora transmitter is NULL");
    B2S_TRY(check_sync(p->ctx, p->cfg.sf, sync0, sync1, "b2s_lora_tx_set_sync_word"));
    p->sync[0] = (unsigned short)sync0;
    p->sync[1] = (unsigned short)sync1;
    return B2S_OK;
}

int32_t b2s_lora_tx_finish(b2s_lora_tx *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "lora transmitter is NULL");
    p->q.finishing = true;
    return B2S_OK;
}

int32_t b2s_lora_tx_pending(const b2s_lora_tx *p, uint64_t *samples) {
    if (!p || !samples) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_lora_tx_pending: NULL argument");
    *samples = p->q.total - p->q.pos;
    return B2S_OK;
}

int32_t b2s_lora_tx_exec(b2s_lora_tx *p, void *d_out, size_t n_out_cap, size_t *produced, int32_t *finished) {
    if (!p || !produced || !finished) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_lora_tx_exec: NULL argument");
    b2s_ctx *ctx = p->ctx;
    *produced = 0;
    const unsigned long long cnt = std::min<unsigned long long>(n_out_cap, p->q.total - p->q.pos);
    if (cnt) {
        if (!d_out || ((uintptr_t)d_out & 7))
            return b2s_fail(ctx, B2S_EINVAL, "b2s_lora_tx_exec: output slice NULL or not 8-byte aligned");
        DeviceGuard g(ctx->device);
        NvtxRange nvtx("b2s_lora_tx_exec");
        const unsigned long long end = p->q.pos + cnt;
        const size_t n_jobs = p->q.open(end);
        const size_t target = 2 * (size_t)std::max(ctx->sm_count, 1);
        const unsigned jpc = (unsigned)std::min<size_t>(kJobs, std::max<size_t>(1, ceil_div(n_jobs, target)));
        ModParams m;
        m.A = p->A.get();
        m.sym = p->sym.b.get();
        m.sym_mask = p->sym.mask();
        m.frames = p->frames.b.get();
        m.frame_mask = p->frames.mask();
        m.f_lo = p->q.f_tail;
        m.n_jobs = (unsigned)n_jobs;
        m.jpc = jpc;
        m.pos = p->q.pos;
        m.cnt = cnt;
        m.out = static_cast<float2 *>(d_out);
        m.N = p->N; m.Q = p->Q; m.pad = p->pad; m.P = p->P; m.extra = p->extra; m.base_len = p->base_len;
        m.sf = (unsigned)p->cfg.sf;
        m.k_up = p->k_up; m.k_down = p->k_down;
        m.sync0 = p->sync[0]; m.sync1 = p->sync[1];
        lora_mod_kernel<<<(unsigned)ceil_div(n_jobs, jpc), kModThreads, kModSmem, ctx->stream>>>(m);
        B2S_CHECK_LAUNCH(ctx);
        p->q.close(end);
        *produced = (size_t)cnt;
    }
    *finished = p->q.finished();
    return B2S_OK;
}

int32_t b2s_lora_tx_drain_bursts(b2s_lora_tx *p, b2s_lora_burst *host, size_t cap, size_t *n) {
    if (!p || !n || (cap && !host)) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_lora_tx_drain_bursts: NULL argument");
    *n = p->q.drain(host, cap);
    return B2S_OK;
}

}  // extern "C"
