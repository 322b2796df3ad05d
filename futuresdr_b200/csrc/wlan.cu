// wlan.cu -- the WLAN transmitter (examples/wlan/src/{mac,encoder,mapper,prefix}.rs and the 64-point inverse Fft of
// bin/tx.rs:44-66) as a device source (DESIGN §4.20).
//
// Encoder, per push, three launches:
//   psdu:   one warp per frame builds the MAC data frame (mac.rs:85-103): header, sequence number << 4, payload and
//           the CRC-32 FCS (lane 0, table-driven, = zlib.crc32).
//   bits:   one CTA per frame.  The scrambled data bits go to shared memory, bit i being the data bit XOR the
//           scrambler's m-sequence at (offset(seed) + i) mod 127, with the 6 tail bits zeroed.  Every coded,
//           punctured and interleaved bit is then an index map onto a 7-bit window of them, so each thread forms whole
//           subcarrier bytes (split_symbols) on its own.  The SIGNAL symbol's 48 BPSK bytes are formed here too.
//   shadow: the bytes a later push's pad bits may read (see below).
// Stale pad bits (encoder.rs keeps `bits` across frames): data bits 16 + 8 psdu onward are whatever the last longer
// frame left there.  The host resolves, from the frame lengths alone, which frame of the push each pad byte comes
// from (a monotonic stack: O(frames + pad bytes)); bytes older than the push come from a device shadow of the
// encoder's 1528 PSDU bytes, which the push then brings up to date.
//
// OFDM exec (the hot path): the stream is cut into tiles of 1024-8192 samples, one CTA each.  A CTA finds its first frame
// by a 32-ary search over the device frame records, writes pads and the sync field as plain stores, and for the
// OFDM symbols its tile touches maps the subcarrier bytes (mapper.rs:23-69) into the 64-entry inputs with the
// inverse fftshift applied on load, runs the library's 64-point Stockham passes exactly as fft.cu's inverse kernel
// does (conj, passes, conj, * sqrtf(1/52)), and writes cyclic prefix, body and window times 0.6 (prefix.rs:57-141).
// A symbol's window reads y_{k-1}[0], so a run of symbols recomputes the one before it.  Every sample is a function
// of its stream position alone: execs never synchronise and any slicing gives the same stream.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "common.cuh"
#include "fft_common.cuh"
#include "tx_common.cuh"

namespace {

using namespace fftk;

constexpr unsigned kMaxPayload = B2S_WLAN_MAX_PAYLOAD;
constexpr unsigned kMaxPsdu = kMaxPayload + 28;                        // header, FCS
constexpr unsigned kPadBytes = 28;                                     // ceil((6 + 215) / 8): tail + pad bits
constexpr unsigned kMaxDataBits = 12384;                               // max over MCS of n_data_bits at kMaxPsdu

// ---- MCS (lib.rs:223-312), indexed by B2S_WLAN_* ------------------------------------------------------------------
__host__ __device__ inline unsigned n_bpsc(int m) { return m < 2 ? 1 : m < 4 ? 2 : m < 6 ? 4 : 6; }
__host__ __device__ inline unsigned n_dbps(int m) { return m == 6 ? 192 : 12 * n_bpsc(m) * ((m & 1) ? 3 : 2); }
__host__ __device__ inline unsigned rate_field(int m) {     // 0x0d 0x0f 0x05 0x07 0x09 0x0b 0x01 0x03
    return (m < 2 ? 0x0d : m < 4 ? 0x05 : m < 6 ? 0x09 : 0x01) | ((m == 6 ? 0 : m & 1) << 1);
}
// 0: rate 1/2, 1: 3/4 (drop i % 6 in {3, 4}), 2: 2/3 (drop i % 4 == 3)   (encoder.rs:55-86)
__host__ __device__ inline int puncturing(int m) { return m == 6 ? 2 : (m & 1); }

// FrameParam::new (lib.rs:323-363): data OFDM symbols of a PSDU
inline unsigned data_symbols(int m, size_t psdu) { return (unsigned)ceil_div(16 + 8 * psdu + 6, n_dbps(m)); }

// ---- generated tables ---------------------------------------------------------------------------------------------
// The scrambler x^7 + x^4 + 1 (encoder.rs:33-53): from state s the output is bit 6 ^ bit 3, shifted in at bit 0.  From
// state 0x7F it runs through all 127 non-zero states; seq is that output (POLARITY[i] = 1 - 2 seq[i]) and offset[s]
// the step at which state s comes up, so a frame scrambled from seed s XORs bit i with seq[(offset[s] + i) % 127].
struct Scrambler {
    unsigned char seq[127];
    unsigned char offset[128];
    constexpr Scrambler() : seq(), offset() {
        unsigned s = 0x7F;
        for (int i = 0; i < 127; ++i) {
            offset[s] = (unsigned char)i;
            const unsigned fb = ((s >> 6) ^ (s >> 3)) & 1u;
            seq[i] = (unsigned char)fb;
            s = ((s << 1) & 0x7Eu) | fb;
        }
    }
};
__constant__ Scrambler kScr = Scrambler();

// the 802.11a short and long training symbols, bins -32..31 (IEEE 802.11-2020 eqs. 17-6, 17-8)
constexpr signed char kShort[64] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, -1, 0, 0, 0, 1, 0, 0, 0, -1, 0, 0, 0, -1, 0,
                                    0, 0, 1, 0, 0, 0, 0, 0, 0, 0, -1, 0, 0, 0, -1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0,
                                    1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0};
constexpr signed char kLong[64] = {0, 0, 0, 0, 0, 0, 1, 1, -1, -1, 1, 1, -1, 1, -1, 1, 1, 1, 1, 1, 1, -1, -1, 1, 1,
                                   -1, 1, -1, 1, 1, 1, 1, 0, 1, -1, -1, 1, 1, -1, 1, -1, 1, -1, -1, -1, -1, -1, 1, 1,
                                   -1, -1, 1, -1, 1, -1, 1, 1, 1, 1, 0, 0, 0, 0, 0};

// SYNC_WORDS (prefix.rs): t[n] = sqrt(1/52) sum_k X[k] e^{2 pi i k n / 64} in f64 (= IFFT(X) 64 sqrt(1/52)), the short
// symbol X = sqrt(13/6) (1 + i) kShort tiled to 160 samples, then the long one as lt[32:] ++ lt ++ lt, sample 160 being
// 0.5 (lt[32] + st[0]); rounded to f32.  The sums are exactly zero wherever the table is: the rounding residue of the
// f64 sums (below 1e-9, against |t| >= 0.02 elsewhere) is snapped to 0.
std::vector<float2> sync_words() {
    const double PI = 3.14159265358979323846264338327950288, c = std::sqrt(13.0 / 6.0);
    auto ifft = [&](const signed char *X, double scale_re, double scale_im, double out[64][2]) {
        for (int n = 0; n < 64; ++n) {
            double re = 0, im = 0;
            for (int i = 0; i < 64; ++i) {
                if (!X[i]) continue;
                const int k = i - 32;
                const double ang = 2.0 * PI * (double)(((k * n) % 64 + 64) % 64) / 64.0;
                const double xr = X[i] * scale_re, xi = X[i] * scale_im;
                re += xr * std::cos(ang) - xi * std::sin(ang);
                im += xr * std::sin(ang) + xi * std::cos(ang);
            }
            if (std::fabs(re) < 1e-9) re = 0;
            if (std::fabs(im) < 1e-9) im = 0;
            out[n][0] = re * std::sqrt(1.0 / 52.0);
            out[n][1] = im * std::sqrt(1.0 / 52.0);
        }
    };
    double st[64][2], lt[64][2];
    ifft(kShort, c, c, st);
    ifft(kLong, 1.0, 0.0, lt);
    std::vector<float2> w(320);
    for (int n = 0; n < 160; ++n) w[n] = make_float2((float)st[n % 64][0], (float)st[n % 64][1]);
    for (int n = 0; n < 160; ++n) {
        const int i = (n + 32) % 64;
        w[160 + n] = make_float2((float)lt[i][0], (float)lt[i][1]);
    }
    w[160] = make_float2((float)(0.5 * (lt[32][0] + st[0][0])), (float)(0.5 * (lt[32][1] + st[0][1])));
    return w;
}

// ---- encoder ------------------------------------------------------------------------------------------------------
struct WFrame {                        // one frame of a push, built on the host
    unsigned long long pay_off;        // its payload in the staged payloads
    unsigned long long psdu_off;       // its PSDU in the PSDU buffer
    unsigned long long sym_abs;        // its SIGNAL symbol (symbol index before the ring mask)
    unsigned psdu;                     // PSDU bytes
    unsigned short seq;                // the sequence number before << 4
    unsigned char seed, mcs;
    int pad_src[kPadBytes];            // PSDU byte psdu + j: byte psdu + j of push frame pad_src[j], or -1: the shadow
};

struct MacAddrs {
    unsigned char a[18];               // src, dst, bss
};

// a subcarrier byte record of the symbol ring; sc[48] is n_bpsc and sc[49] the pilot polarity index in ring records
struct alignas(16) OfdmSym {
    unsigned char sc[64];
};

struct SymOut {                        // where the encoder writes symbol a: base + (a & mask) * stride
    unsigned char *base;
    unsigned long long mask;
    unsigned stride;
    int meta;                          // write n_bpsc and the pilot index (ring records)
};

constexpr int kPsduWarps = 4;

__global__ void __launch_bounds__(kPsduWarps * 32) wlan_psdu_kernel(const unsigned char *pay, const WFrame *frames,
                                                                    unsigned n, MacAddrs mac, unsigned char *psdu) {
    __shared__ unsigned s_crc[256];
    __shared__ unsigned char s_frame[kPsduWarps][kMaxPsdu];
    for (unsigned i = threadIdx.x; i < 256; i += blockDim.x) {       // the reflected CRC-32 table, polynomial 0xEDB88320
        unsigned c = i;
        for (int k = 0; k < 8; ++k) c = (c & 1u) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
        s_crc[i] = c;
    }
    __syncthreads();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned f = blockIdx.x * kPsduWarps + w;
    if (f >= n) return;
    const WFrame fr = frames[f];
    unsigned char *b = s_frame[w];
    const unsigned len = fr.psdu - 4;
    for (unsigned i = lane; i < len; i += 32) {
        unsigned char v;
        if (i < 2) v = i == 0 ? 0x08 : 0x00;                          // frame control 0x0008 LE
        else if (i < 4) v = 0;                                         // duration
        else if (i < 22) v = mac.a[i - 4];
        else if (i < 24) v = (unsigned char)((unsigned)(fr.seq << 4) >> (8 * (i - 22)));
        else v = pay[fr.pay_off + i - 24];
        b[i] = v;
    }
    __syncwarp();
    unsigned crc = 0;
    if (lane == 0) {
        crc = 0xFFFFFFFFu;
        for (unsigned i = 0; i < len; ++i) crc = s_crc[(crc ^ b[i]) & 0xFFu] ^ (crc >> 8);
        crc = ~crc;
    }
    crc = __shfl_sync(~0u, crc, 0);
    for (unsigned i = lane; i < fr.psdu; i += 32)
        psdu[fr.psdu_off + i] = i < len ? b[i] : (unsigned char)(crc >> (8 * (i - len)));
}

// interleave (encoder.rs:88-114): coded bit k of a symbol of n_cbps bits comes from punctured bit second[first[k]]
__device__ __forceinline__ unsigned interleave_src(unsigned k, unsigned cbps, unsigned bpsc) {
    const unsigned s = bpsc / 2 > 1 ? bpsc / 2 : 1;
    const unsigned f = s * (k / s) + (k + 16 * k / cbps) % s;
    return 16 * f - (cbps - 1) * (16 * f / cbps);
}

// the coded bit e (encoded[e], encoder.rs:55-64) of the scrambled bits s: the 7-bit window ending at bit e / 2
__device__ __forceinline__ unsigned coded_bit(const unsigned char *s, unsigned e) {
    const unsigned d = e >> 1;
    unsigned st = 0;
#pragma unroll
    for (int t = 0; t < 7; ++t) st |= (d >= (unsigned)t ? (unsigned)s[d - t] : 0u) << t;
    return __popc(st & ((e & 1u) ? 0117u : 0155u)) & 1u;
}

__global__ void __launch_bounds__(256) wlan_bits_kernel(const WFrame *frames, const unsigned char *psdu,
                                                        const unsigned char *shadow, SymOut out) {
    __shared__ unsigned char s_bits[kMaxDataBits];
    __shared__ unsigned char s_seq[127];
    const WFrame &fr = frames[blockIdx.x];
    const int m = fr.mcs;
    const unsigned bpsc = n_bpsc(m), dbps = n_dbps(m), cbps = 48 * bpsc, p = fr.psdu;
    const unsigned n_sym = (16 + 8 * p + 6 + dbps - 1) / dbps, n_bits = n_sym * dbps;
    const unsigned off = kScr.offset[fr.seed], tail = 16 + 8 * p;
    for (unsigned i = threadIdx.x; i < 127; i += blockDim.x) s_seq[i] = kScr.seq[i];
    __syncthreads();
    for (unsigned i = threadIdx.x; i < n_bits; i += blockDim.x) {
        unsigned bit = 0;
        if (i >= tail && i < tail + 6) {
            s_bits[i] = 0;                                             // tail bits, reset after scrambling
            continue;
        }
        if (i >= 16) {
            const unsigned j = (i - 16) >> 3;
            unsigned byte;
            if (j < p) byte = psdu[fr.psdu_off + j];
            else {                                                     // stale pad byte
                const int src = fr.pad_src[j - p];
                byte = src >= 0 ? psdu[frames[src].psdu_off + j] : (j < kMaxPsdu ? shadow[j] : 0u);
            }
            bit = (byte >> ((i - 16) & 7)) & 1u;
        }
        s_bits[i] = (unsigned char)(bit ^ s_seq[(off + i) % 127]);
    }
    __syncthreads();
    const int pm = puncturing(m);
    // data symbols 1..n_sym: byte q of the frame's data is subcarrier q % 48 of symbol 1 + q / 48
    for (unsigned q = threadIdx.x; q < 48 * n_sym; q += blockDim.x) {
        const unsigned i = q / 48, c = q - i * 48;
        unsigned v = 0;
        for (unsigned k = 0; k < bpsc; ++k) {
            const unsigned pb = i * cbps + interleave_src(c * bpsc + k, cbps, bpsc);
            const unsigned e = pm == 0 ? pb : pm == 1 ? (pb / 4) * 6 + (pb % 4 == 3 ? 5 : pb % 4) : (pb / 3) * 4 + pb % 3;
            v |= coded_bit(s_bits, e) << k;
        }
        unsigned char *rec = out.base + ((fr.sym_abs + 1 + i) & out.mask) * out.stride;
        rec[c] = (unsigned char)v;
        if (out.meta && c == 0) {
            rec[48] = (unsigned char)bpsc;
            rec[49] = (unsigned char)((i + 1) % 127);
        }
    }
    // SIGNAL (mapper.rs:23-69): rate MSB first, reserved 0, 12-bit length LSB first, even parity, 6 zero tail bits;
    // rate-1/2 coded and interleaved as one BPSK symbol of 48 coded bits
    if (threadIdx.x < 48) {
        const unsigned rate = rate_field(m);
        unsigned char sig[24];
        unsigned par = 0;
        for (int i = 0; i < 24; ++i) {
            unsigned b = 0;
            if (i < 4) b = (rate >> (3 - i)) & 1u;
            else if (i >= 5 && i < 17) b = (p >> (i - 5)) & 1u;
            if (i < 17) par ^= b;
            sig[i] = (unsigned char)(i == 17 ? par : b);
        }
        const unsigned c = threadIdx.x;
        unsigned char *rec = out.base + (fr.sym_abs & out.mask) * out.stride;
        rec[c] = (unsigned char)coded_bit(sig, interleave_src(c, 48, 1));
        if (out.meta && c == 0) {
            rec[48] = 1;
            rec[49] = 0;
        }
    }
}

__global__ void wlan_shadow_kernel(const int *src, const WFrame *frames, const unsigned char *psdu,
                                   unsigned char *shadow) {
    for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < kMaxPsdu; j += gridDim.x * blockDim.x)
        if (src[j] >= 0) shadow[j] = psdu[frames[src[j]].psdu_off + j];
}

// The host half of one encode: frame table, PSDU offsets and the pad byte sources of frames from a fresh shadow
// position on (Enc.bits as the shadow holds it).  shadow_src[j] is the frame whose byte j the shadow takes after the
// push, or -1 to keep it.
struct EncPlan {
    std::vector<WFrame> frames;
    std::vector<int> shadow_src;
    size_t pay_bytes = 0, psdu_bytes = 0, n_sym = 0;
};

int32_t check_mcs(b2s_ctx *ctx, int32_t m, const char *what) {
    if (m < 0 || m > 7) return b2s_fail(ctx, B2S_EINVAL, "%s: MCS %d is not 0..7", what, m);
    return B2S_OK;
}

// lengths / mcs (HOST, mcs NULL or -1: default_mcs); seed, seq: the first frame's
int32_t plan_encode(b2s_ctx *ctx, const size_t *lengths, const int32_t *mcs, size_t n, int32_t default_mcs,
                    unsigned seed, unsigned seq, unsigned long long sym0, EncPlan &pl, const char *what) {
    pl.frames.resize(n);
    pl.shadow_src.assign(kMaxPsdu, -1);
    std::vector<int> stack;            // frames of the push whose bytes Enc.bits still holds: PSDUs decrease upward
    for (size_t f = 0; f < n; ++f) {
        if (lengths[f] > kMaxPayload)
            return b2s_fail(ctx, B2S_EINVAL, "%s: a payload of %zu bytes (at most %u)", what, lengths[f], kMaxPayload);
        const int32_t m = mcs && mcs[f] != -1 ? mcs[f] : default_mcs;
        B2S_TRY(check_mcs(ctx, m, what));
        WFrame &w = pl.frames[f];
        w.pay_off = pl.pay_bytes;
        w.psdu_off = pl.psdu_bytes;
        w.sym_abs = sym0 + pl.n_sym;
        w.psdu = (unsigned)lengths[f] + 28;
        w.seq = (unsigned short)((seq + f) % 4096);
        w.seed = (unsigned char)((seed - 1 + f) % 127 + 1);
        w.mcs = (unsigned char)m;
        const unsigned n_sym = data_symbols(m, w.psdu);
        while (!stack.empty() && pl.frames[stack.back()].psdu <= w.psdu) stack.pop_back();
        // byte j >= psdu: the topmost stacked frame longer than j
        const unsigned hi = std::min<unsigned>(w.psdu + kPadBytes, (n_sym * n_dbps(m) - 16 + 7) / 8);
        unsigned j = w.psdu;
        for (size_t s = stack.size(); s-- > 0 && j < hi;)
            for (; j < std::min(pl.frames[stack[s]].psdu, hi); ++j) w.pad_src[j - w.psdu] = stack[s];
        for (; j < w.psdu + kPadBytes; ++j) w.pad_src[j - w.psdu] = -1;
        stack.push_back((int)f);
        pl.pay_bytes += lengths[f];
        pl.psdu_bytes += w.psdu;
        pl.n_sym += 1 + n_sym;
    }
    unsigned j = 0;
    for (size_t s = stack.size(); s-- > 0;)
        for (; j < pl.frames[stack[s]].psdu; ++j) pl.shadow_src[j] = stack[s];
    return B2S_OK;
}

// the three encode launches; frames, psdu and shadow_src are device copies of the plan's
int32_t launch_encode(b2s_ctx *ctx, const EncPlan &pl, const unsigned char *pay, const WFrame *frames,
                      const MacAddrs &mac, unsigned char *psdu, unsigned char *shadow, const int *shadow_src,
                      const SymOut &out) {
    const size_t n = pl.frames.size();
    if (!n) return B2S_OK;
    wlan_psdu_kernel<<<(unsigned)ceil_div(n, kPsduWarps), kPsduWarps * 32, 0, ctx->stream>>>(pay, frames, (unsigned)n,
                                                                                             mac, psdu);
    B2S_CHECK_LAUNCH(ctx);
    wlan_bits_kernel<<<(unsigned)n, 256, 0, ctx->stream>>>(frames, psdu, shadow, out);
    B2S_CHECK_LAUNCH(ctx);
    if (shadow_src) {
        wlan_shadow_kernel<<<(unsigned)ceil_div(kMaxPsdu, 256), 256, 0, ctx->stream>>>(shadow_src, frames, psdu, shadow);
        B2S_CHECK_LAUNCH(ctx);
    }
    return B2S_OK;
}

// ---- OFDM exec ------------------------------------------------------------------------------------------------------
constexpr int kExecThreads = 256;
constexpr FftGeom kG = fft_geom(6, kExecThreads);      // 4 threads per transform, 64 transforms per batch
constexpr unsigned kTileMax = 8192;                    // stream samples per CTA: a large exec
constexpr unsigned kTileMin = 1024;                    // a small exec still spreads over every SM

struct WTxFrame {                      // device record of one queued frame
    unsigned long long start, sym_abs; // stream index of its first sample; its SIGNAL symbol
    unsigned n_ofdm;                   // OFDM symbols: SIGNAL + data
    unsigned pad_;
};

struct ExecParams {
    const OfdmSym *sym;
    unsigned long long sym_mask;
    const WTxFrame *frames;
    unsigned long long frame_mask, f_lo;
    unsigned n_frames;                 // frames that [pos, pos + cnt) touches, from f_lo on
    unsigned long long pos, cnt;
    unsigned tile;                     // stream samples per CTA
    float2 *out;
    const float2 *tw;
    const float2 *sync;                // SYNC_WORDS
    unsigned long long pad_front, tail; // tail = max(pad_tail, 1)
    float norm;                        // sqrtf(1 / 52)
};

// Modulation::map (lib.rs:66-175): levels formed in f32, i.e. (a * LEVEL) rounded once
__device__ __forceinline__ float level(unsigned bits, unsigned nb) {
    if (nb == 1) return (bits & 1u) ? 0.70710677f : -0.70710677f;                 // FRAC_1_SQRT_2
    if (nb == 2) {
        const float a = (bits & 2u) ? ((bits & 1u) ? 1.0f : -1.0f) : ((bits & 1u) ? 3.0f : -3.0f);
        return __fmul_rn(a, 0.31622776601683794f);
    }
    const unsigned h = (bits >> 1) & 3u;                                          // -7 7 -1 1 -5 5 -3 3
    const float mag = h == 0 ? 7.0f : h == 1 ? 1.0f : h == 2 ? 5.0f : 3.0f;
    return __fmul_rn((bits & 1u) ? mag : -mag, 0.1543033499620919f);
}
__device__ __forceinline__ float2 constellation(unsigned b, unsigned bpsc) {
    switch (bpsc) {
    case 1: return make_float2(b ? 1.0f : -1.0f, 0.0f);
    case 2: return make_float2(level(b, 1), level(b >> 1, 1));
    case 4: return make_float2(level(b, 2), level(b >> 2, 2));
    default: return make_float2(level(b, 3), level(b >> 3, 3));
    }
}

// Mapper::map, output subcarrier c of a symbol record
__device__ __forceinline__ float2 subcarrier(const unsigned char *rec, int c) {
    if (c < 6 || c > 58 || c == 32) return make_float2(0.0f, 0.0f);
    if (c == 11 || c == 25 || c == 39 || c == 53) {
        const float pol = kScr.seq[rec[49]] ? -1.0f : 1.0f;                 // POLARITY[index % 127]
        return c == 53 ? make_float2(-pol, -0.0f) : make_float2(pol, 0.0f);
    }
    const int d = c - (c < 11 ? 6 : c < 25 ? 7 : c < 32 ? 8 : c < 39 ? 9 : c < 53 ? 10 : 11);
    return constellation(rec[d], rec[48]);
}

__device__ __forceinline__ float2 scale06(float2 v) { return make_float2(__fmul_rn(v.x, 0.6f), __fmul_rn(v.y, 0.6f)); }
__device__ __forceinline__ float2 window(float2 a, float2 b) {     // 0.5 * (a + b)
    return make_float2(__fmul_rn(0.5f, __fadd_rn(a.x, b.x)), __fmul_rn(0.5f, __fadd_rn(a.y, b.y)));
}

__global__ void __launch_bounds__(kExecThreads, 5) wlan_exec_kernel(const ExecParams a) {
    __shared__ __align__(16) float2 s_y[kG.fpb * kG.np];
    __shared__ OfdmSym s_rec[kG.fpb];
    __shared__ unsigned long long s_f;
    const unsigned long long t0 = a.pos + (unsigned long long)blockIdx.x * a.tile;
    const unsigned long long t1 = min(t0 + a.tile, a.pos + a.cnt);
    // the last frame starting at or before t0, by warp 0
    if (threadIdx.x < 32) {
        const unsigned long long f = tx_first_frame(a.frames, a.frame_mask, a.f_lo, a.n_frames, t0);
        if (threadIdx.x == 0) s_f = f;
    }
    __syncthreads();
    const int t = threadIdx.x % kG.t, fl = threadIdx.x / kG.t;
    float2 *sm = s_y + fl * kG.np;
    for (unsigned long long fi = s_f; fi < a.n_frames; ++fi) {
        const WTxFrame fr = a.frames[(a.f_lo + fi) & a.frame_mask];
        const unsigned long long d0 = a.pad_front + 320, len = fr.n_ofdm, end = d0 + 80 * len + a.tail;
        if (fr.start >= t1) break;
        const unsigned long long ra = max(t0, fr.start) - fr.start, rb = min(t1, fr.start + end) - fr.start;
        float2 *o = a.out + (fr.start - a.pos);
        const unsigned long long sa = d0, sb = d0 + 80 * len + 1;       // samples that read a transform
        // pads and the sync field: plain stores
        auto plain = [&](unsigned long long r) {
            return (r >= a.pad_front && r < d0) ? scale06(a.sync[r - a.pad_front]) : make_float2(0.0f, 0.0f);
        };
        store_range<kExecThreads>(o, ra, min(rb, sa), plain);
        store_range<kExecThreads>(o, max(ra, sb), rb, plain);
        const unsigned long long qa = max(ra, sa), qb = min(rb, sb);
        if (qa >= qb) continue;
        const unsigned long long ka = (qa - d0) / 80, kb = (qb - 1 - d0) / 80;   // kb may be len: the tail window
        for (unsigned long long kw = ka; kw <= kb;) {
            const unsigned long long c0 = kw == 0 ? 0 : kw - 1;
            const unsigned nt = (unsigned)min((unsigned long long)kG.fpb, min(kb, len - 1) - c0 + 1);
            unsigned long long kend = c0 + nt - 1;
            if (kend == len - 1 && kb >= len) kend = len;
            __syncthreads();                                           // the previous batch's samples are written
            for (unsigned i = threadIdx.x; i < nt * 4; i += kExecThreads)
                reinterpret_cast<uint4 *>(s_rec)[i] =
                    reinterpret_cast<const uint4 *>(a.sym + ((fr.sym_abs + c0 + i / 4) & a.sym_mask))[i % 4];
            __syncthreads();
            const unsigned char *rec = s_rec[fl < (int)nt ? fl : 0].sc;
            // fft.cu's inverse kernel with shift and norm: buff[k] = in[(k + 32) % 64], conj, passes, conj, * norm
            fft_passes<6, kG.t, Tw::Table>(
                [&](int idx) {
                    float2 x = subcarrier(rec, (idx + 32) & 63);
                    x.y = -x.y;
                    return x;
                },
                [&](int idx, float2 y) {
                    y.y = -y.y;
                    y.x *= a.norm; y.y *= a.norm;
                    sm[pad(idx)] = y;
                },
                sm, a.tw, t, false, true);
            // samples [wa, wb) from the transforms in slots 0..nt-1; indices relative to slot 0's first sample fit 32 bits
            const unsigned long long base = d0 + 80 * c0;
            const unsigned u0 = (unsigned)(max(qa, d0 + 80 * kw) - base), u1 = (unsigned)(min(qb, d0 + 80 * (kend + 1)) - base);
            const unsigned last = (unsigned)(len - c0);                // the slot of the tail window sample, if any
            store_range<kExecThreads>(o + base, u0, u1, [&](unsigned u) {
                const unsigned slot = u / 80, s = u - 80 * slot;
                const float2 *y = s_y + slot * kG.np;
                float2 v;
                if (s == 0) {
                    const float2 prev = slot == 0 ? a.sync[256] : y[-kG.np];   // slot 0 is symbol 0 here
                    v = slot == last ? window(make_float2(0.0f, 0.0f), prev) : window(y[pad(48)], prev);
                } else {
                    v = s < 16 ? y[pad(48 + s)] : y[pad(s - 16)];
                }
                return scale06(v);
            });
            kw = kend + 1;
        }
    }
}

}  // namespace

struct b2s_wlan_tx {
    b2s_ctx *ctx = nullptr;
    MacAddrs mac{};
    int32_t default_mcs = 0;
    unsigned long long pad_front = 0, pad_tail = 0;
    unsigned seed = 1, seq = 0;
    float norm = 1.0f;
    Buf<float2> tw, sync;
    Buf<unsigned char> shadow;         // the encoder's PSDU bytes as Enc.bits holds them after the last push
    DevRing<OfdmSym> sym;
    DevRing<WTxFrame> frames;
    Buf<unsigned char> pay, psdu;      // the payloads and PSDUs of the last push
    Buf<WFrame> enc;
    Buf<int> shadow_src;
    TxQueue<b2s_wlan_burst> q;

    unsigned long long frame_len(unsigned n_ofdm) const {
        return pad_front + 320 + 80ull * n_ofdm + std::max<unsigned long long>(pad_tail, 1);
    }
};

namespace {
int32_t check_frame(b2s_ctx *ctx, int32_t mcs, size_t psdu_len, const char *what) {
    B2S_TRY(check_mcs(ctx, mcs, what));
    if (psdu_len > kMaxPsdu) return b2s_fail(ctx, B2S_EINVAL, "%s: a PSDU of %zu bytes (at most %u)", what, psdu_len,
                                             kMaxPsdu);
    return B2S_OK;
}
}  // namespace

extern "C" {

int32_t b2s_wlan_frame_param(int32_t mcs, size_t psdu_len, size_t *n_symbols, size_t *n_data_bits, size_t *n_pad) {
    if (!n_symbols || !n_data_bits || !n_pad) return b2s_fail(nullptr, B2S_EINVAL, "b2s_wlan_frame_param: NULL argument");
    B2S_TRY(check_frame(nullptr, mcs, psdu_len, "b2s_wlan_frame_param"));
    *n_symbols = data_symbols(mcs, psdu_len);
    *n_data_bits = *n_symbols * n_dbps(mcs);
    *n_pad = *n_data_bits - (16 + 8 * psdu_len + 6);
    return B2S_OK;
}

int32_t b2s_wlan_encode(b2s_ctx *ctx, const uint8_t src[6], const uint8_t dst[6], const uint8_t bss[6],
                        uint32_t sequence_number, uint32_t scrambler_seed, const uint8_t *d_payloads,
                        const size_t *lengths, const int32_t *mcs, size_t n_frames, uint8_t *d_symbols,
                        size_t symbols_cap, size_t *n_symbols) {
    if (!ctx || !n_symbols || !src || !dst || !bss || (n_frames && (!lengths || !mcs)))
        return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_encode: NULL argument");
    *n_symbols = 0;
    if (scrambler_seed < 1 || scrambler_seed > 127)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_encode: scrambler seed %u is not 1..127", scrambler_seed);
    if (sequence_number > 4095)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_encode: sequence number %u is not 0..4095", sequence_number);
    EncPlan pl;
    B2S_TRY(plan_encode(ctx, lengths, mcs, n_frames, -1, scrambler_seed, sequence_number, 0, pl, "b2s_wlan_encode"));
    if (pl.pay_bytes && !d_payloads) return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_encode: NULL payloads");
    if (pl.n_sym > symbols_cap)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_encode: %zu symbols do not fit %zu", pl.n_sym, symbols_cap);
    if (pl.n_sym && !d_symbols) return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_encode: NULL symbols");
    if (!n_frames) return B2S_OK;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_wlan_encode");
    MacAddrs mac;
    std::copy(src, src + 6, mac.a);
    std::copy(dst, dst + 6, mac.a + 6);
    std::copy(bss, bss + 6, mac.a + 12);
    // frame table, PSDUs and a zero shadow (a fresh Enc) in stream-ordered memory, freed after the kernels
    const size_t fb = n_frames * sizeof(WFrame);
    void *d_w = nullptr;
    B2S_CUDA(ctx, cudaMallocAsync(&d_w, fb + pl.psdu_bytes + kMaxPsdu, ctx->stream));
    unsigned char *d_psdu = static_cast<unsigned char *>(d_w) + fb, *d_shadow = d_psdu + pl.psdu_bytes;
    B2S_CUDA(ctx, cudaMemcpyAsync(d_w, pl.frames.data(), fb, cudaMemcpyHostToDevice, ctx->stream));
    B2S_CUDA(ctx, cudaMemsetAsync(d_shadow, 0, kMaxPsdu, ctx->stream));
    const int32_t rc = launch_encode(ctx, pl, d_payloads, static_cast<const WFrame *>(d_w), mac, d_psdu, d_shadow,
                                     nullptr, SymOut{d_symbols, ~0ull, 48, 0});
    B2S_CUDA(ctx, cudaFreeAsync(d_w, ctx->stream));
    B2S_TRY(rc);
    *n_symbols = pl.n_sym;
    return B2S_OK;
}

int32_t b2s_wlan_tx_create(b2s_ctx *ctx, const uint8_t src[6], const uint8_t dst[6], const uint8_t bss[6],
                           int32_t default_mcs, size_t pad_front, size_t pad_tail, b2s_wlan_tx **out) {
    if (!ctx || !out || !src || !dst || !bss) return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_tx_create: NULL argument");
    *out = nullptr;
    B2S_TRY(check_mcs(ctx, default_mcs, "b2s_wlan_tx_create"));
    if (pad_front > 0xFFFFFFFFull || pad_tail > 0xFFFFFFFFull)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_tx_create: pads %zu / %zu above 2^32 - 1", pad_front, pad_tail);
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_wlan_tx> p(new b2s_wlan_tx());
    p->ctx = ctx;
    std::copy(src, src + 6, p->mac.a);
    std::copy(dst, dst + 6, p->mac.a + 6);
    std::copy(bss, bss + 6, p->mac.a + 12);
    p->default_mcs = default_mcs;
    p->pad_front = pad_front;
    p->pad_tail = pad_tail;
    p->norm = std::sqrt(1.0f / 52.0f);                       // (1.0f32 / 52.0).sqrt() (tx.rs:60)
    const std::vector<float2> tw = twiddle_table(64), sw = sync_words();
    B2S_TRY(p->tw.upload(ctx, tw.data(), tw.size(), "b2s_wlan_tx_create: twiddles"));
    B2S_TRY(p->sync.upload(ctx, sw.data(), sw.size(), "b2s_wlan_tx_create: sync words"));
    B2S_TRY(p->shadow.alloc(ctx, kMaxPsdu, "b2s_wlan_tx_create: pad shadow"));
    B2S_CUDA(ctx, cudaMemsetAsync(p->shadow.get(), 0, kMaxPsdu, ctx->stream));
    B2S_TRY(p->shadow_src.alloc(ctx, kMaxPsdu, "b2s_wlan_tx_create: shadow sources"));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));       // the host tables die here
    *out = p.release();
    return B2S_OK;
}

void b2s_wlan_tx_destroy(b2s_wlan_tx *p) { PlanDeleter<b2s_wlan_tx>()(p); }

int32_t b2s_wlan_tx_reset(b2s_wlan_tx *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "wlan transmitter is NULL");
    p->q.reset();
    p->seed = 1;
    p->seq = 0;
    DeviceGuard g(p->ctx->device);
    B2S_CUDA(p->ctx, cudaMemsetAsync(p->shadow.get(), 0, kMaxPsdu, p->ctx->stream));
    return B2S_OK;
}

int32_t b2s_wlan_tx_push(b2s_wlan_tx *p, const uint8_t *payloads, const size_t *lengths, const int32_t *mcs,
                         size_t n_frames) {
    if (!p || (n_frames && !lengths)) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_wlan_tx_push: NULL argument");
    b2s_ctx *ctx = p->ctx;
    EncPlan pl;
    B2S_TRY(plan_encode(ctx, lengths, mcs, n_frames, p->default_mcs, p->seed, p->seq, p->q.s_head, pl,
                        "b2s_wlan_tx_push"));
    if (pl.pay_bytes && !payloads) return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_tx_push: NULL payloads");
    if (!n_frames) return B2S_OK;
    std::vector<WTxFrame> rec(n_frames);
    std::vector<TxHostFrame> hf(n_frames);
    unsigned long long start = p->q.total;
    for (size_t i = 0; i < n_frames; ++i) {
        const WFrame &w = pl.frames[i];
        const unsigned n_ofdm = 1 + data_symbols(w.mcs, w.psdu);
        rec[i] = WTxFrame{start, w.sym_abs, n_ofdm, 0};
        hf[i] = TxHostFrame{start, p->frame_len(n_ofdm), w.sym_abs};
        start += hf[i].len;
    }
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("b2s_wlan_tx_push");
    B2S_TRY(p->frames.make_room(ctx, p->q.f_tail, p->q.f_head, n_frames, "b2s_wlan_tx_push: frame records"));
    B2S_TRY(p->sym.make_room(ctx, p->q.s_tail, p->q.s_head, pl.n_sym, "b2s_wlan_tx_push: symbols"));
    B2S_TRY(p->pay.reserve(ctx, std::max<size_t>(pl.pay_bytes, 1), "b2s_wlan_tx_push: payloads"));
    B2S_TRY(p->psdu.reserve(ctx, pl.psdu_bytes, "b2s_wlan_tx_push: PSDUs"));
    B2S_TRY(p->enc.reserve(ctx, n_frames, "b2s_wlan_tx_push: frame table"));
    if (pl.pay_bytes)
        B2S_CUDA(ctx, cudaMemcpyAsync(p->pay.get(), payloads, pl.pay_bytes, cudaMemcpyHostToDevice, ctx->stream));
    B2S_CUDA(ctx, cudaMemcpyAsync(p->enc.get(), pl.frames.data(), n_frames * sizeof(WFrame), cudaMemcpyHostToDevice,
                                  ctx->stream));
    B2S_CUDA(ctx, cudaMemcpyAsync(p->shadow_src.get(), pl.shadow_src.data(), kMaxPsdu * sizeof(int),
                                  cudaMemcpyHostToDevice, ctx->stream));
    B2S_TRY(p->frames.put(ctx, p->q.f_head, rec.data(), n_frames));
    B2S_TRY(launch_encode(ctx, pl, p->pay.get(), p->enc.get(), p->mac, p->psdu.get(), p->shadow.get(),
                          p->shadow_src.get(),
                          SymOut{reinterpret_cast<unsigned char *>(p->sym.b.get()), p->sym.mask(), 64, 1}));
    p->q.append(hf, pl.n_sym);
    p->seed = (unsigned)((p->seed - 1 + n_frames) % 127 + 1);
    p->seq = (unsigned)((p->seq + n_frames) % 4096);
    return B2S_OK;
}

int32_t b2s_wlan_tx_finish(b2s_wlan_tx *p) {
    if (!p) return b2s_fail(nullptr, B2S_EINVAL, "wlan transmitter is NULL");
    p->q.finishing = true;
    return B2S_OK;
}

int32_t b2s_wlan_tx_pending(const b2s_wlan_tx *p, uint64_t *samples) {
    if (!p || !samples) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_wlan_tx_pending: NULL argument");
    *samples = p->q.total - p->q.pos;
    return B2S_OK;
}

int32_t b2s_wlan_tx_exec(b2s_wlan_tx *p, void *d_out, size_t n_out_cap, size_t *produced, int32_t *finished) {
    if (!p || !produced || !finished) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_wlan_tx_exec: NULL argument");
    b2s_ctx *ctx = p->ctx;
    *produced = 0;
    const unsigned long long cnt = std::min<unsigned long long>(n_out_cap, p->q.total - p->q.pos);
    if (cnt) {
        if (!d_out || ((uintptr_t)d_out & 7))
            return b2s_fail(ctx, B2S_EINVAL, "b2s_wlan_tx_exec: output slice NULL or not 8-byte aligned");
        DeviceGuard g(ctx->device);
        NvtxRange nvtx("b2s_wlan_tx_exec");
        const unsigned long long end = p->q.pos + cnt;
        ExecParams a;
        a.sym = p->sym.b.get();
        a.sym_mask = p->sym.mask();
        a.frames = p->frames.b.get();
        a.frame_mask = p->frames.mask();
        a.f_lo = p->q.f_tail;
        a.n_frames = (unsigned)p->q.open(end);
        a.pos = p->q.pos;
        a.cnt = cnt;
        a.out = static_cast<float2 *>(d_out);
        a.tw = p->tw.get();
        a.sync = p->sync.get();
        a.pad_front = p->pad_front;
        a.tail = std::max<unsigned long long>(p->pad_tail, 1);
        a.norm = p->norm;
        // at least ~8 CTAs per SM where the exec is large enough; every tile size gives the same samples
        const size_t want = round_up(ceil_div(cnt, 8 * (size_t)std::max(ctx->sm_count, 1)), kTileMin);
        a.tile = (unsigned)std::min<size_t>(kTileMax, want);
        wlan_exec_kernel<<<(unsigned)ceil_div(cnt, a.tile), kExecThreads, 0, ctx->stream>>>(a);
        B2S_CHECK_LAUNCH(ctx);
        p->q.close(end);
        *produced = (size_t)cnt;
    }
    *finished = p->q.finished();
    return B2S_OK;
}

int32_t b2s_wlan_tx_drain_bursts(b2s_wlan_tx *p, b2s_wlan_burst *host, size_t cap, size_t *n) {
    if (!p || !n || (cap && !host)) return b2s_fail(p ? p->ctx : nullptr, B2S_EINVAL, "b2s_wlan_tx_drain_bursts: NULL argument");
    *n = p->q.drain(host, cap);
    return B2S_OK;
}

}  // extern "C"
