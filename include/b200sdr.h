/*
 * b200sdr.h -- C ABI of the H100-native streaming-DSP backend for FutureSDR's
 * FIR / decimator / resampler / FFT / Apply / PfbArbResampler hot path.
 *
 * The reference (FutureSDR, Rust) has no FFI for this path: its boundary is a set of Rust
 * traits.  Every entry point below names the reference interface it replaces (file:line is
 * relative to the FutureSDR tree).  INTEGRATION.md shows the Rust `extern "C"` block and the
 * `impl futuredsp::Filter` / `impl Kernel` shims a maintainer would add on top of this header.
 *
 * Conventions
 *   - every function returns int32_t: 0 = B2S_OK, <0 = B2S_E*; b2s_last_error() gives text.
 *     No exception crosses the boundary, no torch/CUDA type appears in a signature
 *     (a CUDA stream is passed as void*).
 *   - handles are opaque; a handle is used by one caller at a time (thread-compatible),
 *     different handles may be used concurrently.
 *   - Complex<f32> is interleaved {re, im} (num_complex is repr(C)); item counts are in
 *     ITEMS (samples), never bytes, exactly like the Rust slices they replace.
 *   - *_exec calls take DEVICE pointers, are asynchronous and ordered on the context's
 *     stream; the (consumed, produced, status) triple is a pure function of the sizes and is
 *     returned immediately.  *_host calls take HOST pointers and return when the output is
 *     in host memory (they are the literal drop-in for `Filter::filter(&[In], &mut [Out])`).
 */
#ifndef B200SDR_H
#define B200SDR_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_VERSION 100 /* 0.1.0 */

/* ---- status codes ---------------------------------------------------------------------- */
#define B2S_OK            0
#define B2S_EINVAL       (-1) /* bad argument (the reference would panic/assert)            */
#define B2S_ECUDA        (-2) /* CUDA runtime error; sticky, see b2s_last_error             */
#define B2S_ENOMEM       (-3)
#define B2S_EAGAIN       (-4) /* ring: no buffer available right now (not an error)         */
#define B2S_EUNSUPPORTED (-5) /* combination the reference supports but this build does not */
#define B2S_ESTATE       (-6) /* slot/ring used out of order                                */
#define B2S_ETIMEOUT     (-7) /* a cross-GPU flag wait gave up (the peer never published)   */

/* futuredsp::ComputationStatus  (crates/futuredsp/src/lib.rs:33-45) */
#define B2S_INSUFFICIENT_INPUT  0
#define B2S_INSUFFICIENT_OUTPUT 1
#define B2S_BOTH_SUFFICIENT     2

/* sample x tap kinds = the Filter impls that exist in futuredsp
 * (fir.rs:206-276, decimating_fir.rs:99-300, polyphase_resampling_fir.rs:126-167) */
typedef enum {
    B2S_F32_F32 = 0, /* f32 samples, f32 taps                 */
    B2S_C32_F32 = 1, /* Complex<f32> samples, f32 taps        */
    B2S_C32_C32 = 2, /* Complex<f32> samples, Complex<f32> taps */
    B2S_F64_F64 = 3  /* f64 samples, f64 taps (fir.rs:217-226; plan with b2s_fir_plan_f64_f64) */
} b2s_kind;

/* FIR algorithm selection (no reference equivalent; AUTO picks by tap count / kind) */
typedef enum {
    B2S_ALGO_AUTO   = 0,
    B2S_ALGO_DIRECT = 1, /* CUDA-core register-blocked direct form (any kind, any decimation) */
    B2S_ALGO_TENSOR = 2, /* wgmma block-Toeplitz GEMM, split-bf16 (real taps, 16..257, decim divides 128).
                          * Numerics: operands are split into bf16 hi + lo and three of the four partial products are
                          * summed in FP32: ~2^-18 rms per product, worst case ~3e-5 of ||taps||_1 max|x| when EVERY
                          * product errs the same way (constant taps on constant input -- AUTO keeps constant tap
                          * vectors on DIRECT).  Non-finite input: a NaN/Inf sample at index i makes outputs of the
                          * 128-sample blocks whose issued K-range contains it non-finite (all inside [i-K, i+131],
                          * K = 128*ceil((ntaps+127)/128), a superset of the reference's [i-ntaps+1, i]); all other
                          * outputs are unaffected and no finite output is ever wrong.  f32 DENORMAL samples may count as
                          * zero (tensor-core operands may be flushed to zero).  Streams that may carry
                          * non-finite samples and need the reference's exact propagation: use B2S_ALGO_DIRECT. */
    B2S_ALGO_FFT    = 3, /* overlap-save FFT convolution (c32 samples, 64..2049 taps, decim == 1).
                          * Numerics: block b of a call reads the NF = 4096 inputs x_b = x[s, s+NF) (zeros past the end),
                          * s = b*V, and writes outputs [s, s+V), V = NF-(ntaps-1), through two single-precision FFTs and
                          * H = FFT(taps)/NF rounded to f32.  Error: |y_k - exact| <= 8 * 2^-24 * log2(NF) *
                          * (||taps||_2 * rms(x_b) + rms(c_b)), c_b the block's circular output (rms <= max|G| rms(x_b)):
                          * it follows the block's INPUT, not y -- a stopband output carries an input-sized error.
                          * Non-finite input: a NaN/Inf sample at index i makes every output of every block whose window
                          * holds i non-finite (all inside [i-NF+1, i+NF-ntaps], a superset of the reference's
                          * [i-ntaps+1, i]; the last block reads its whole window, also samples past what its outputs
                          * need); all other outputs are unaffected.  Finite range: outputs are finite while
                          * 4096 * max|x| * max(1, ||taps||_1) < 2^128; past it each output is within the bound or
                          * non-finite, never a wrong finite value.  Tiny input: below max|x| ~ 2^-100 the products
                          * X.H reach the subnormal range and the bound holds plus ||taps||_1 * 2^-126, down to
                          * denormal-only input.  Streams that need the reference's exact propagation: use
                          * B2S_ALGO_DIRECT. */
    B2S_ALGO_SCAN   = 4  /* IIR only (b2s_iir_set_algo): single-pass chained scan, see b2s_iir below;
                          * b2s_fir_set_algo rejects it */
} b2s_algo;

typedef struct b2s_ctx    b2s_ctx;
typedef struct b2s_fir    b2s_fir;
typedef struct b2s_resamp b2s_resamp;
typedef struct b2s_pfbarb b2s_pfbarb;
typedef struct b2s_fft    b2s_fft;
typedef struct b2s_apply  b2s_apply;
typedef struct b2s_ring   b2s_ring;
typedef struct b2s_slot   b2s_slot;

/* ---- context (replaces runtime::buffer::vulkan::Instance, buffer/vulkan/mod.rs:45-153) -- */
int32_t     b2s_version(void);
/* b2s_ctx_create: the context creates (and owns) a non-blocking stream.
 * b2s_ctx_create_on_stream: `stream` is a cudaStream_t owned by the caller (e.g. torch's current
 * stream; 0 / NULL means the legacy default stream) and all work is ordered on it. */
int32_t     b2s_ctx_create(int device, b2s_ctx **out);
int32_t     b2s_ctx_create_on_stream(int device, void *stream, b2s_ctx **out);
void        b2s_ctx_destroy(b2s_ctx *ctx);
const char *b2s_last_error(const b2s_ctx *ctx); /* ctx may be NULL: last global error       */
int32_t     b2s_ctx_sync(b2s_ctx *ctx);         /* ≙ awaiting the fence, blocks/vulkan.rs:157-162 */
void       *b2s_ctx_stream(b2s_ctx *ctx);
int32_t     b2s_ctx_sm_count(b2s_ctx *ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t    b2s_ctx_launch_count(const b2s_ctx *ctx);
/* device + pinned bytes currently held by the objects created on this context (plans, sub-plans, rings and their
   exec-time workspaces); the context's own status word and host-pipeline workspace are not counted */
uint64_t    b2s_ctx_bytes_held(const b2s_ctx *ctx);

/* device / pinned-host memory (≙ Instance::create_buffer, buffer/vulkan/mod.rs:132) */
int32_t b2s_malloc(b2s_ctx *ctx, size_t bytes, void **dptr);
int32_t b2s_free(b2s_ctx *ctx, void *dptr);
int32_t b2s_host_alloc(b2s_ctx *ctx, size_t bytes, void **hptr); /* pinned */
int32_t b2s_host_free(b2s_ctx *ctx, void *hptr);
int32_t b2s_memcpy_h2d(b2s_ctx *ctx, void *dptr, const void *hptr, size_t bytes); /* async */
int32_t b2s_memcpy_d2h(b2s_ctx *ctx, void *hptr, const void *dptr, size_t bytes); /* async */

/* ---- FIR plans (≙ FirFilter::new fir.rs:39-46, DecimatingFirFilter::new decimating_fir.rs:41-49)
 * taps: ntaps items of f32 (or interleaved Complex<f32> for B2S_C32_C32), in the SAME order the
 * reference takes them (the filter applies them reversed, fir.rs:84); copied at creation.
 * decim == 1 gives FirFilter, decim > 1 DecimatingFirFilter. */
int32_t b2s_fir_plan(b2s_ctx *ctx, b2s_kind kind, const float *taps, size_t ntaps, size_t decim,
                     b2s_fir **out);
int32_t b2s_fir_plan_f32_f32(b2s_ctx *ctx, const float *taps, size_t ntaps, size_t decim, b2s_fir **out);
int32_t b2s_fir_plan_c32_f32(b2s_ctx *ctx, const float *taps, size_t ntaps, size_t decim, b2s_fir **out);
int32_t b2s_fir_plan_c32_c32(b2s_ctx *ctx, const float *taps, size_t ntaps, size_t decim, b2s_fir **out);
/* f64 samples x f64 taps (fir.rs:217-226, decimating_fir.rs:117-130): plain CUDA-core form, un-fused multiply/add in
 * tap order -- bit-identical to the stable-Rust loop; b2s_fir_exec / b2s_fir_exec_hist take f64 items. */
int32_t b2s_fir_plan_f64_f64(b2s_ctx *ctx, const double *taps, size_t ntaps, size_t decim, b2s_fir **out);
void    b2s_fir_destroy(b2s_fir *f);
size_t  b2s_fir_length(const b2s_fir *f);           /* ≙ Filter::length, lib.rs:65-67 */
int32_t b2s_fir_set_algo(b2s_fir *f, b2s_algo algo);
int32_t b2s_fir_get_algo(const b2s_fir *f);         /* the algorithm AUTO resolved to */

/* ≙ Filter::filter (lib.rs:58-64; cores fir.rs:52-91, decimating_fir.rs:53-95): device slices.
 * Elements of d_out beyond *produced are left unspecified, as in the reference. */
int32_t b2s_fir_exec(b2s_fir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                     size_t *consumed, size_t *produced, int32_t *status);
/* Same contract on the LOGICAL slice  d_hist[0..n_hist) ++ d_in[0..n_in):  the history a FIR block keeps in front
 * of new samples (blocks/fir.rs:49 min_items, slab.rs:370-398) handed over as a separate pointer, so that it can live
 * in another ring slot -- or in ANOTHER GPU's memory (SURVEY 8e: the last ntaps-1 samples of the left neighbour's
 * shard; `d_hist` is then a peer address from b2s_ipc_open / b2s_peer_enable).  On the tensor path the kernel's TMA
 * loader fetches the history itself (over NVLink for peer memory): one launch, no copy, no host synchronisation.
 * Other paths copy it into the n_hist items in FRONT of d_in, which must therefore be writable scratch of the same
 * allocation (a ring slot's halo region; b2s_ring_create(..., halo_items >= n_hist, ...)).
 * Optional cross-GPU handshake `hs` (NULL = none; every flag pointer inside may be NULL as well), all system scope,
 * see b2s_flag_*:  publish: *publish_flag = publish_value is stored when the call starts executing -- "my chunk
 * (everything queued on this context before the call) is in HBM", what the right neighbour waits for;  wait: before
 * reading the history the device spins until *wait_flag >= wait_value;  done: *done_flag = done_value is stored
 * once the history has been read, so its owner may overwrite it.  On the tensor path all three happen INSIDE the FIR
 * kernel (no extra launch). */
typedef struct b2s_handshake {
    uint32_t       *publish_flag; uint32_t publish_value;
    const uint32_t *wait_flag;    uint32_t wait_value;
    uint32_t       *done_flag;    uint32_t done_value;
} b2s_handshake;
int32_t b2s_fir_exec_hist(b2s_fir *f, const void *d_hist, size_t n_hist, const void *d_in, size_t n_in,
                          void *d_out, size_t n_out_cap, const b2s_handshake *hs, size_t *consumed, size_t *produced,
                          int32_t *status);
/* Same contract with host slices (pageable or pinned): chunked H2D -> kernel -> D2H pipeline
 * through an internal device ring; returns after the last D2H completed. */
int32_t b2s_fir_filter_host(b2s_fir *f, const void *h_in, size_t n_in, void *h_out, size_t n_out_cap,
                            size_t *consumed, size_t *produced, int32_t *status);

/* ---- rational polyphase resampler (≙ PolyphaseResamplingFir, polyphase_resampling_fir.rs:42-124)
 * kinds B2S_F32_F32 and B2S_C32_F32 (the only impls, :126-167); ntaps % interp == 0 (:56).  interp > 4096,
 * decim > 65536 or ntaps > 2^20 is refused at plan time (B2S_EUNSUPPORTED); every plan that is accepted executes. */
int32_t b2s_resamp_plan(b2s_ctx *ctx, b2s_kind kind, const float *taps, size_t ntaps, size_t interp,
                        size_t decim, b2s_resamp **out);
void    b2s_resamp_destroy(b2s_resamp *r);
size_t  b2s_resamp_length(const b2s_resamp *r);
int32_t b2s_resamp_exec(b2s_resamp *r, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                        size_t *consumed, size_t *produced, int32_t *status);

/* ---- PfbArbResampler (≙ src/blocks/pfb/arb_resampler.rs:90-231; Complex<f32> only).
 * Stateful like the block: one exec == one Kernel::work call (window fill first, :199-215). */
int32_t b2s_pfbarb_plan_c32(b2s_ctx *ctx, const float *taps, size_t ntaps, size_t num_filters,
                            float rate, b2s_pfbarb **out);
void    b2s_pfbarb_destroy(b2s_pfbarb *p);
int32_t b2s_pfbarb_reset(b2s_pfbarb *p);
/* Host-only diagnostic: the timing recurrence (update_timing_state :130-140, `tau -= 1.0` :184-186) is periodic; this
 * returns the period in input items and the outputs it produces (0, 0 when no cycle shorter than 2^25 items starts at
 * tau = 0 -- such plans replay the recurrence on the host per call).  Needs no device. */
int32_t b2s_pfbarb_period(float rate, size_t num_filters, uint64_t *period_items, uint64_t *outputs_per_period);
int32_t b2s_pfbarb_exec(b2s_pfbarb *p, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                        size_t *consumed, size_t *produced, int32_t *call_again);

/* ---- FFT (≙ Fft::with_options, src/blocks/fft.rs:66-121, and Fft::work :160-221) ---------
 * inverse: FftDirection; fft_shift, normalize as in with_options (has_normalize = Option::is_some).
 * One exec processes m = floor(min(n_in, n_out_cap)/n)*n items (no 32-FFT cap: the cap only
 * splits work across calls, fft.rs:171).
 * Lengths: any n >= 2 like rustfft.  Powers of two <= 16384 and other lengths <= 8192 run as ONE pass through shared
 * memory (Stockham / fused Bluestein: 16 B/sample of HBM traffic); larger ones -- powers of two up to 2^26, other
 * lengths up to 2^24 -- use the four-step algorithm through HBM on top of two shared-memory plans (five passes;
 * the plan owns 2 n / 4 M items of scratch).  Changing the length = destroy + create (fft.rs:124-151's handler). */
int32_t b2s_fft_plan_c32(b2s_ctx *ctx, size_t n, int32_t inverse, int32_t fft_shift,
                         int32_t has_normalize, float normalize, b2s_fft **out);
void    b2s_fft_destroy(b2s_fft *f);
size_t  b2s_fft_length(const b2s_fft *f);
int32_t b2s_fft_exec(b2s_fft *f, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                     size_t *consumed, size_t *produced);

/* ---- Apply (≙ src/blocks/apply.rs:100-131).  The reference takes an arbitrary Rust closure;
 * the device version is a closed catalogue of the closures used on the path. */
typedef enum {
    B2S_OP_SCALE_F32     = 0, /* f32 -> f32: x * param          (tests/vulkan.rs:16-27, blocks/wgpu.rs:22-32) */
    B2S_OP_SCALE_C32     = 1, /* c32 -> c32: x * param                                                       */
    B2S_OP_QUAD_DEMOD    = 2, /* c32 -> f32: arg(x[n] * conj(x[n-1])), stateful (examples/fm-receiver/src/main.rs:99-104) */
    B2S_OP_NORM_SQR      = 3, /* c32 -> f32: re^2 + im^2        (examples/spectrum/src/bin/cpu.rs)            */
    B2S_OP_QUAD_DEMOD_C32 = 4, /* c32 -> c32 {re: phase, im: 0}: demod packed for PfbArbResampler (SURVEY §7) */
    B2S_OP_EXP_F32       = 5, /* f32 -> f32: exp(x)            (examples/vulkan/src/main.rs:17-29)            */
    B2S_OP_MAG_C32       = 6, /* c32 -> f32: sqrt(re^2 + im^2)                                               */
    B2S_OP_LOG10_F32     = 7, /* f32 -> f32: param * log10(x)   (spectrum dB stage)                           */
    B2S_OP_DC_BLOCK_F32  = 8, /* f32 -> f32: s = (1 - param) * s + param * x; y = x - s, stateful, s starts at 0
                               * (the one-pole DC blocker of examples/zigbee/src/bin/rx.rs:66-74 and
                               * examples/keyfob/src/main.rs:62-68).  param must be finite (B2S_EINVAL otherwise).
                               * A sequential recurrence: bit-exact under any slicing, one CTA per call. */
    B2S_OP_SLICE_F32_U8  = 9, /* f32 -> u8: x > 0 ? 1 : 0 (NaN and +-0 give 0), the keyfob receiver's slicer
                               * (examples/keyfob/src/main.rs:73-75).  The input slice must be 4-byte aligned, the
                               * output may start at any byte; the slices must not overlap (B2S_EINVAL otherwise). */
    B2S_OP_DIV_C32       = 10, /* c32 -> c32: x / param, each part divided (num_complex Complex / f32).  With
                               * B2S_OP_SCALE_C32 by 2 in front it is the SSB transmitter's file level
                               * `v * 2.0 / 0.0001` (examples/ssb/transmit.rs:125) bit for bit. */
    B2S_OP_C32_TO_I16_IQ = 11  /* c32 -> i16 pairs: out[2j] = (re * param * 32767.0) as i16, out[2j+1] the same of im
                               * (examples/ssb/transmit.rs:109-112, param 0.9): products rounded in that order, then
                               * Rust's `as i16` -- truncation toward zero, saturation to [-32768, 32767], NaN -> 0.
                               * TWO output items per input item: consumed = min(n_in, n_out_cap / 2) and
                               * produced = 2 * consumed (ApplyNM<1, 2>, src/blocks/applynm.rs:109-117).  The input
                               * must be 8-byte aligned and the output 2-byte aligned (any i16 item start); the
                               * slices must not overlap (B2S_EINVAL otherwise). */
} b2s_op;
int32_t b2s_apply_create(b2s_ctx *ctx, b2s_op op, float param, b2s_apply **out);
void    b2s_apply_destroy(b2s_apply *a);
int32_t b2s_apply_reset(b2s_apply *a); /* closure state back to its initial value */
/* m = min(n_in, n_out_cap) items are processed (apply.rs:109), except by B2S_OP_C32_TO_I16_IQ (above).
 * Element-wise ops may run in place (d_in == d_out);
 * the stateful demodulators (B2S_OP_QUAD_DEMOD*) need disjoint slices (B2S_EINVAL otherwise).  Their output is
 * the arg of the f32 product with libm atan2's special values, within 4e-7 rad: (+-inf, +-inf) gives +-pi/4 or
 * +-3pi/4, signed zeros give +-0 or +-pi, and a NaN part gives NaN. */
int32_t b2s_apply_exec(b2s_apply *a, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                       size_t *consumed, size_t *produced);

/* ---- Rotator + XlatingFir helper (≙ futuredsp::Rotator, crates/futuredsp/src/rotator.rs:13-48;
 * XlatingFir = DecimatingFirFilter with band-pass Complex<f32> taps + Rotator at the output rate,
 * src/blocks/xlating_fir.rs:72-126 -- build the FIR with b2s_fir_plan(B2S_C32_C32, bpf, n, decim)).
 * The rotator keeps its phase across calls exactly like the reference object. */
typedef struct b2s_rotator b2s_rotator;
int32_t b2s_rotator_create(b2s_ctx *ctx, float phase_incr, b2s_rotator **out);
void    b2s_rotator_destroy(b2s_rotator *r);
int32_t b2s_rotator_reset(b2s_rotator *r);
/* ≙ Rotator::rotate (:32-47); d_in == d_out is rotate_inplace (:24-29). n = min(n_in, n_out_cap). */
int32_t b2s_rotator_exec(b2s_rotator *r, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                         size_t *processed, int32_t *status);
/* xlating_fir.rs:80-86 and :97-99: band-pass taps (2*ntaps floats) and the rotator's phase increment */
int32_t b2s_xlating_taps(const float *taps, size_t ntaps, float offset, float sample_rate, size_t decimation,
                         float *bpf_interleaved, float *rotator_phase_incr);

/* ---- Oscillator mixers: the Apply closures of the SSB example that carry an oscillator,
 *      `let mut osc = Complex32::new(1.0, 0.0); ... osc *= shift; f(v, osc)` with
 *      shift = Complex32::from_polar(1.0, phase_incr) -- the Rotator's recurrence, replayed by the same code, so every
 *      op is bit-identical to the reference closure under any slicing of the stream (DESIGN §4.18). */
typedef enum {
    B2S_MIX_ROTATE_C32       = 0, /* c32 -> c32: v * osc (examples/ssb/transmit.rs:102-107); == b2s_rotator_exec     */
    B2S_MIX_ROTATE_SCALE_C32 = 1, /* c32 -> c32: v * osc * param, each part scaled (receive.rs:58-66, param 0.0001)   */
    B2S_MIX_WEAVER_F32       = 2  /* c32 -> f32: param * (v.re * osc.re + v.im * osc.im) (receive.rs:73-83, param 0.5) */
} b2s_mix_op;
typedef struct b2s_mixer b2s_mixer;
int32_t b2s_mixer_create(b2s_ctx *ctx, b2s_mix_op op, float phase_incr, float param, b2s_mixer **out);
void    b2s_mixer_destroy(b2s_mixer *m);
int32_t b2s_mixer_reset(b2s_mixer *m); /* osc back to 1 + 0i (the closure's initial state) */
/* m = min(n_in, n_out_cap) samples (apply.rs:109); consumed = produced = m.  The input must be 8-byte aligned and the
 * output aligned to its item.  The ROTATE ops may run in place (d_in == d_out, no other overlap); the Weaver needs
 * disjoint slices (B2S_EINVAL otherwise).  Like b2s_rotator_exec, a call only waits when the stream has outrun the
 * host replay of the recurrence. */
int32_t b2s_mixer_exec(b2s_mixer *m, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                       size_t *consumed, size_t *produced);

/* ---- PfbChannelizer (≙ src/blocks/pfb/channelizer.rs:88-223; SURVEY §8f-2): polyphase FIR bank +
 * N-point inverse FFT per output vector.  Stateful like the block: one exec == one Kernel::work
 * call (window fill first; note the reference does not consume on the call that completes the fill).
 * d_out is channel-major: output stream ch starts at d_out + ch * out_stride items. */
typedef struct b2s_chan b2s_chan;
int32_t b2s_chan_plan_c32(b2s_ctx *ctx, size_t num_channels, const float *taps, size_t ntaps, float oversample_rate,
                          b2s_chan **out);
void    b2s_chan_destroy(b2s_chan *c);
size_t  b2s_chan_decimation(const b2s_chan *c);
int32_t b2s_chan_exec(b2s_chan *c, const void *d_in, size_t n_in, void *d_out, size_t out_stride, size_t n_out_cap,
                      size_t *consumed, size_t *produced_per_channel, int32_t *call_again);

/* ---- PfbSynthesizer (≙ src/blocks/pfb/synthesizer.rs:52-144; SURVEY §8f-2): N-point inverse FFT per
 * input vector + polyphase FIR bank, N outputs per vector.  d_in is channel-major (stream w starts at
 * d_in + w * in_stride items), n_in = the shortest input slice.  One exec == one Kernel::work call.
 * Power-of-two banks up to 256 channels with <= 32 taps per arm run as ONE fused kernel in the steady state. */
typedef struct b2s_synth b2s_synth;
int32_t b2s_synth_plan_c32(b2s_ctx *ctx, size_t num_channels, const float *taps, size_t ntaps, b2s_synth **out);
void    b2s_synth_destroy(b2s_synth *s);
int32_t b2s_synth_exec(b2s_synth *s, const void *d_in, size_t in_stride, size_t n_in, void *d_out, size_t n_out_cap,
                       size_t *consumed_per_channel, size_t *produced);

/* ---- MovingAvg<WIDTH> (≙ src/blocks/moving_avg.rs:24-116; SURVEY §8f-3, tail of the spectrum pipe
 * Fft(shift) -> |x|^2 -> MovingAvg).  f32 items; state (avg[WIDTH], chunk counter) kept on the device. */
typedef struct b2s_mavg b2s_mavg;
int32_t b2s_mavg_create(b2s_ctx *ctx, size_t width, float decay_factor, size_t history_size, b2s_mavg **out);
void    b2s_mavg_destroy(b2s_mavg *m);
int32_t b2s_mavg_exec(b2s_mavg *m, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                      size_t *consumed, size_t *produced);

/* ---- IirFilter (≙ crates/futuredsp/src/iir.rs:33-178, the core of src/blocks/iir.rs): StatefulFilter::filter.
 * y = sum_j b[j] * x[k + n_b - 1 - j] + sum_j a[j] * memory[j] (PLUS sign on the a-term, b[0] multiplies the newest
 * sample), then memory shifts and memory[0] = y.  Before the first output `memory` is filled with the stream's first
 * n_a INPUT samples (memory[0] = x[0]); those are not consumed and a call that fills memory returns (0, 0).  Each call
 * produces n = min(n_in - n_b + 1, n_out_cap) outputs and consumes as many; the status is the reference's (:166-177).
 * memory and the fill count live in the plan (on the device): calls are stream-ordered and never synchronise.
 * n_b == 0 is B2S_EINVAL (the reference asserts, :132); n_a and n_b are each limited to 2048.  Input and output
 * slices must not overlap.
 * Algorithms:
 *   B2S_ALGO_DIRECT  one thread runs the recurrence with un-fused IEEE multiply/add in the reference's order:
 *                    bit-identical to the reference for f32 and f64, denormals and non-finite values included (NaN
 *                    payloads aside).  About 5-12 Msamples/s (one GPU thread walks the recurrence).
 *   B2S_ALGO_SCAN    f32 only; 1 <= n_a <= 8, n_b <= 64 and a stable filter: ||A^(2^20)|| < 1e-3 in f64 (A: the
 *                    companion matrix of a), i.e. max|pole| < 1 - 6.6e-6.  Blocked scan of the state recurrence with
 *                    decoupled look-back across 4096-output tiles, 8 B/sample of HBM traffic.
 *                    Numerics: each run of 16 outputs is re-computed with the reference's operations from a start
 *                    state that the scan evaluates in a different order (f32 FMA, matrix powers rounded from f64),
 *                    so outputs are not bit-identical to the reference.  With G = ||h||_1 + sum_j ||g_j||_1 (h: the
 *                    impulse response, g_j: the zero-input response to memory e_j), the error against the exact
 *                    (f64) recurrence is within max(1e-5 G max|x|, 2 x the reference's own f32 error), and the
 *                    distance to the reference within 1e-5 G max|x| + the reference's own f32 error.  Near the unit
 *                    circle on DC input the f32 reference itself drifts by ~eps/(1-r); the scan stays closer to the
 *                    exact value there.  A NaN/Inf input at index i makes every output from i - n_b + 1 on
 *                    non-finite, exactly the reference's set (0 * NaN = NaN carries it through the state).
 *                    A look-back wait that exceeds 4 s gives up and b2s_ctx_sync reports B2S_ETIMEOUT.
 *   B2S_ALGO_AUTO    SCAN when the plan is admitted, otherwise DIRECT; a pure-FIR plan (n_a == 0) runs on a FIR plan
 *                    with taps = b (the same sum, added oldest sample first) and b2s_iir_get_algo reports the FIR's
 *                    algorithm.  The choice depends on the plan only, never on the call size. */
typedef struct b2s_iir b2s_iir;
int32_t b2s_iir_plan_f32(b2s_ctx *ctx, const float *a_taps, size_t n_a, const float *b_taps, size_t n_b, b2s_iir **out);
int32_t b2s_iir_plan_f64(b2s_ctx *ctx, const double *a_taps, size_t n_a, const double *b_taps, size_t n_b,
                         b2s_iir **out);
void    b2s_iir_destroy(b2s_iir *f);
size_t  b2s_iir_length(const b2s_iir *f);            /* ≙ StatefulFilter::length: n_b */
int32_t b2s_iir_set_algo(b2s_iir *f, b2s_algo algo); /* AUTO, DIRECT or SCAN; SCAN on a plan it does not admit: EUNSUPPORTED */
int32_t b2s_iir_get_algo(const b2s_iir *f);          /* the algorithm AUTO resolved to */
int32_t b2s_iir_exec(b2s_iir *f, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                     size_t *consumed, size_t *produced, int32_t *status);

/* ---- SignalSource (≙ src/blocks/signal_source/mod.rs:29-227, SignalSourceBuilder :110-227) with its fixed-point NCO
 * (fxpt_nco.rs:3-43) and FixedPointPhase (fxpt_phase.rs:8-99).  A source: no input, each exec fills the WHOLE output
 * slice (mod.rs:94-104) and the block never finishes.  The phase is a wrapping 32-bit integer, so output k of a call
 * is f(phase0 + k inc) * amplitude with nothing carried between samples: the device output is bit-identical to the
 * reference at any stream length, signed zeros from a zero or negative amplitude included.  NaN outputs (NaN amplitude,
 * or 0 * inf) carry the bit patterns of the reference's f32 multiply on x86-64: the amplitude's NaN quieted, or the
 * default NaN 0xFFC00000.
 *   create: phase0 = FixedPointPhase::new(initial_phase), inc = FixedPointPhase::new(((2 PI) frequency) / sample_rate),
 *           all in f32 (mod.rs:130-133).  Like the reference nothing is validated: sample_rate == 0, NaN or inf give
 *           whatever FixedPointPhase::new makes of them (Rust's saturating `as i32`, NaN -> 0).
 *   waves:  f32       COS cos(phase), SIN sin(phase), SQUARE (value < 0 ? 1 : 0)
 *           Complex32 COS and SIN both (cos, sin) (mod.rs:175-199); SQUARE maps value >> 30 as -2 -> (1,0),
 *           -1 -> (1,1), 0 -> (0,1), 1 -> (0,0) (:213-221); each times amplitude.
 *   exec:   writes n_out_cap items at d_out (4-byte aligned; no other alignment needed), *produced = n_out_cap, then
 *           advances the phase by n_out_cap steps.  Phase and increment live in the plan on the host: calls are
 *           stream-ordered and never synchronise.  set_amplitude applies from the next exec. */
typedef enum { B2S_WAVE_COS = 0, B2S_WAVE_SIN = 1, B2S_WAVE_SQUARE = 2 } b2s_wave;
typedef struct b2s_sigsrc b2s_sigsrc;
int32_t b2s_sigsrc_create(b2s_ctx *ctx, b2s_wave wave, int32_t complex_items, float frequency, float sample_rate,
                          float amplitude, float initial_phase, b2s_sigsrc **out);
void    b2s_sigsrc_destroy(b2s_sigsrc *s);
int32_t b2s_sigsrc_set_amplitude(b2s_sigsrc *s, float amplitude);      /* ≙ SignalSource::set_amplitude (:71-73) */
/* the NCO's current phase (the next sample's FixedPointPhase::value) and its increment */
int32_t b2s_sigsrc_phase(const b2s_sigsrc *s, int32_t *value, int32_t *inc);
int32_t b2s_sigsrc_exec(b2s_sigsrc *s, void *d_out, size_t n_out_cap, size_t *produced);
/* Host-only mirrors of the public FixedPointPhase (need no device): new(x) (fxpt_phase.rs:75-82) and sin() / cos()
 * (:85-98) of a phase value, from the same sine table the kernel uses. */
int32_t b2s_fxpt_phase_new(float x, int32_t *value);
int32_t b2s_fxpt_sin_cos(int32_t value, float *sin_out, float *cos_out);

/* ---- fused spectrum pipe (SURVEY §8f-3): Fft::with_options(n, Forward, fft_shift, None) -> Apply(|x|^2) ->
 * MovingAvg<n>::new(decay_factor, history_size) [-> log10_scale * log10(.) when log10_scale != 0] of
 * examples/spectrum/src/bin/cpu.rs:21-28 in ONE pass over the samples: 8 B/sample in, n floats per `history_size`
 * frames out (the three separate blocks above move 32 B/sample through HBM).  Stateful like MovingAvg (avg[], i).
 * The moving average is evaluated as a blocked scan, so values agree with the sequential f32 reference to rounding
 * (~1e-6 relative), not bit for bit -- use b2s_fft + b2s_apply + b2s_mavg where bit equality matters.
 * n: power of two, 32..8192.  consumed counts Complex<f32> items, produced counts f32 items. */
typedef struct b2s_spectrum b2s_spectrum;
int32_t b2s_spectrum_plan(b2s_ctx *ctx, size_t n, int32_t fft_shift, float decay_factor, size_t history_size,
                          float log10_scale, b2s_spectrum **out);
void    b2s_spectrum_destroy(b2s_spectrum *s);
int32_t b2s_spectrum_reset(b2s_spectrum *s);
int32_t b2s_spectrum_exec(b2s_spectrum *s, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                          size_t *consumed, size_t *produced);

/* ---- device-resident buffer ring (≙ buffer/vulkan/{h2d,d2h}.rs + circuit.rs + slab.rs history)
 * n_slots buffers of `halo_items + chunk_items` items each stay in HBM; ownership of a slot
 * moves source-edge -> GPU block(s) -> sink-edge -> back (circuit), exactly like
 * vulkan::Buffer (h2d.rs:161-232, d2h.rs:66-74, :270-299).  Each slot has pinned host staging
 * for the H2D / D2H edges when with_host_staging != 0. */
int32_t b2s_ring_create(b2s_ctx *ctx, size_t item_bytes, size_t chunk_items, size_t halo_items,
                        int32_t n_slots, int32_t with_host_staging, b2s_ring **out);
void    b2s_ring_destroy(b2s_ring *r);
/* ≙ H2DWriter: pop an empty buffer from `inbound` (h2d.rs:178-197); B2S_EAGAIN if none */
int32_t b2s_ring_acquire_empty(b2s_ring *r, b2s_slot **slot);
/* ≙ H2DWriter::produce -> outbound.push + notify (h2d.rs:199-232).  from_host != 0 first
 * enqueues the pinned->device copy of valid_items. */
int32_t b2s_ring_submit_full(b2s_ring *r, b2s_slot *slot, size_t valid_items, int32_t from_host);
/* ≙ H2DReader::buffers() / D2HReader (h2d.rs:276, d2h.rs:247-268); B2S_EAGAIN if none */
int32_t b2s_ring_acquire_full(b2s_ring *r, b2s_slot **slot, size_t *valid_items);
/* ≙ D2HReader::consume -> buffer back to the circuit start (d2h.rs:270-299) */
int32_t b2s_ring_release(b2s_ring *r, b2s_slot *slot);
/* slab.rs:370-398: copy the unconsumed tail (`tail_items` <= halo_items) of `from` in front of
 * `to`'s data so the next block sees contiguous history. */
int32_t b2s_ring_carry_halo(b2s_ring *r, const b2s_slot *from, size_t from_valid, size_t tail_items,
                            b2s_slot *to);
void   *b2s_slot_device_ptr(const b2s_slot *slot); /* first data item; halo lives just below   */
void   *b2s_slot_host_ptr(const b2s_slot *slot);   /* pinned staging (NULL without staging)    */
size_t  b2s_slot_halo_valid(const b2s_slot *slot); /* items of history currently in front      */
int32_t b2s_slot_fetch_to_host(b2s_slot *slot, size_t items); /* async D2H into staging + event */
int32_t b2s_slot_wait(b2s_slot *slot);             /* host wait on the slot's event            */
size_t  b2s_ring_free_slots(const b2s_ring *r);
size_t  b2s_ring_full_slots(const b2s_ring *r);
/* geometry of the ring's single device allocation, for exporting it to a peer process (b2s_ipc_export):
 * a peer addresses slot i's first data item at  peer_base + b2s_ring_slot_offset(i)  and the ring's two u32
 * counters {ready, consumed} at  peer_base + b2s_ring_flags_offset(). */
void   *b2s_ring_base(const b2s_ring *r);
size_t  b2s_ring_bytes(const b2s_ring *r);
size_t  b2s_ring_slot_offset(const b2s_ring *r, int32_t slot_index);
size_t  b2s_ring_flags_offset(const b2s_ring *r);
int32_t b2s_slot_index(const b2s_slot *slot);

/* ---- cross-GPU plumbing of a sharded stream (SURVEY 8e; no reference equivalent -- FutureSDR is single-device).
 * One process per GPU: export a device allocation (d_base = pointer returned by b2s_malloc or b2s_ring_base) as an
 * opaque 64-byte handle, ship the handle to the neighbour by any means (torch.distributed, a pipe), and map it
 * there.  One process driving several GPUs uses b2s_peer_enable instead and passes raw pointers. */
#define B2S_IPC_HANDLE_BYTES 64
int32_t b2s_ipc_export(b2s_ctx *ctx, void *d_base, uint8_t handle[B2S_IPC_HANDLE_BYTES]);
int32_t b2s_ipc_open(b2s_ctx *ctx, const uint8_t handle[B2S_IPC_HANDLE_BYTES], void **d_peer);
int32_t b2s_ipc_close(b2s_ctx *ctx, void *d_peer);
int32_t b2s_peer_enable(b2s_ctx *ctx, int32_t peer_device);
/* Stream-ordered system-scope flags (u32 counters in device memory, local or peer):
 * set = release store after everything queued before it; wait = the stream stalls until *flag >= value (wrap-safe),
 * giving up after 4 s (b2s_ctx_sync then returns B2S_ETIMEOUT).  b2s_flag_read is a blocking host read. */
int32_t b2s_flag_set(b2s_ctx *ctx, uint32_t *d_flag, uint32_t value);
int32_t b2s_flag_wait(b2s_ctx *ctx, const uint32_t *d_flag, uint32_t value);
int32_t b2s_flag_read(b2s_ctx *ctx, const uint32_t *d_flag, uint32_t *value);
int32_t b2s_memcpy_d2d(b2s_ctx *ctx, void *dst, const void *src, size_t bytes); /* async, any two devices */
int32_t b2s_memset(b2s_ctx *ctx, void *dst, int32_t byte, size_t bytes);         /* async */

/* ---- stream plumbing of branching flowgraphs: Combine (src/blocks/combine.rs:102-136), Split (split.rs:95-126),
 * StreamDuplicator (stream_duplicator.rs:66-93) and StreamDeinterleaver (stream_deinterleaver.rs:61-97).  Stateless
 * context-level calls: (consumed, produced) is a pure function of the sizes, returned immediately; the kernels run
 * asynchronously on the context's stream and allocate nothing.  The reference's closures are a closed catalogue here,
 * each evaluated with un-fused IEEE f32 operations in the Rust expression's order: outputs are bit-identical to the
 * reference (NaN payloads aside).  Slices need 4-byte alignment only; any offset and any length (0 and 1 included)
 * work.  An output may coincide exactly with an input of the same item size (in place) or be disjoint from it;
 * any other overlap is B2S_EINVAL.  A NULL slice is B2S_EINVAL when the call would process an item. */
typedef enum {
    B2S_COMBINE_ADD_F32 = 0,       /* f32, f32 -> f32: a + b                      (tests/combine.rs)   */
    B2S_COMBINE_SUB_F32 = 1,       /* f32, f32 -> f32: i1 - i2                    (examples/m17)       */
    B2S_COMBINE_MUL_F32 = 2,       /* f32, f32 -> f32: a * b                      (examples/cw)        */
    B2S_COMBINE_CONJ_MUL_C32 = 3,  /* c32, c32 -> c32: a * b.conj()               (examples/wlan rx)   */
    B2S_COMBINE_MAG_DIV_C32_F32 = 4, /* c32, f32 -> f32: a.norm() / b; norm = glibc hypotf (wlan rx)   */
    B2S_COMBINE_TO_C32 = 5,        /* f32, f32 -> c32: Complex32::new(i, q)       (examples/ssb USB)   */
    B2S_COMBINE_TO_C32_NEG_Q = 6   /* f32, f32 -> c32: Complex32::new(i, q * -1.0) (examples/ssb LSB)  */
} b2s_combine_op;
/* m = min(n_in0, n_in1, n_out_cap) items of each input are consumed and m produced (combine.rs:114-125) */
int32_t b2s_combine_exec(b2s_ctx *ctx, b2s_combine_op op, const void *d_in0, size_t n_in0, const void *d_in1,
                         size_t n_in1, void *d_out, size_t n_out_cap, size_t *consumed, size_t *produced);
typedef enum {
    B2S_SPLIT_RE_IM = 0,           /* c32 -> (f32 re, f32 im)                     (tests/split.rs)     */
    B2S_SPLIT_DUP_F32 = 1          /* f32 -> (v, v)                               (examples/ssb)       */
} b2s_split_op;
/* m = min(n_in, n_out_cap) (split.rs:106-119); n_out_cap is the smaller of the two output slices */
int32_t b2s_split_exec(b2s_ctx *ctx, b2s_split_op op, const void *d_in, size_t n_in, void *d_out0, void *d_out1,
                       size_t n_out_cap, size_t *consumed, size_t *produced);
/* One launch, the input read once, items of item_bytes = 4 or 8 (f32, Complex32, f64).  d_outs is a HOST array of
 * n_outs device pointers; n_out_cap is the smallest free space over the outputs.
 *   deinterleave == 0  StreamDuplicator: out_k[j] = in[j], m = min(n_in, n_out_cap), consumed = produced = m.
 *   deinterleave != 0  StreamDeinterleaver: out_k[j] = in[j n_outs + k] over whole groups only,
 *                      m = min(n_out_cap, n_in / n_outs), consumed = m n_outs, produced = m (per output).
 * The output pointers travel in the kernel's parameter block: n_outs > 256 is B2S_EUNSUPPORTED.  Outputs must not
 * overlap the input or each other. */
int32_t b2s_fanout_exec(b2s_ctx *ctx, int32_t deinterleave, size_t item_bytes, const void *d_in, size_t n_in,
                        void *const *d_outs, size_t n_outs, size_t n_out_cap, size_t *consumed, size_t *produced);

/* ---- the WLAN and M17 receivers' MovingAverage (≙ examples/wlan/src/moving_average.rs:44-107, f32 and Complex32,
 * output = sum; examples/m17/src/moving_average.rs:20-81, f32, output = sum / 4800.0).  Not MovingAvg (b2s_mavg).
 * One reference work() call: while pad > 0 (pad starts at len - 1) it writes m = min(pad, n_out) zeros and consumes
 * nothing, with call_again = m < n_out; afterwards it produces m = min(4000, (n_in + 1) - len (saturating), n_out)
 * window sums, each a strict-order f32 running sum that restarts at the call (sum = fold of x[0 .. len-1] from -0.0
 * for f32, from (+0, +0) for Complex32; then sum += x[i+len-1], out[i] = sum [/ divisor], sum -= x[i]), consumes m,
 * and is finished iff the input is finished and m == (n_in + 1) - len (saturating).  The outputs depend on where the
 * calls fall, so the device reproduces them bit for bit given the same sequence of calls (NaN payloads aside).
 *   create: complex_items as in b2s_sigsrc_create; len == 0 and a divisor with complex_items are B2S_EINVAL.
 *   exec:   emulates the calls the reference makes back to back on what is left of the slices -- the remaining pad,
 *           then runs of up to 4000 outputs -- until a call makes no progress or max_calls calls have run
 *           (max_calls == 0: no limit; 1: exactly one work() call).  *calls counts the emulated calls, the last
 *           one included; *call_again and *done are that call's call_again and its m == (rem_in + 1) - len, which
 *           the caller ANDs with input.finished().  The only state is pad, kept on the host: calls are
 *           stream-ordered and never synchronise.  Slices need 4-byte alignment only; an output overlapping the
 *           input it reads is B2S_EINVAL.
 *   reset:  pad back to len - 1. */
typedef struct b2s_boxavg b2s_boxavg;
int32_t b2s_boxavg_create(b2s_ctx *ctx, int32_t complex_items, size_t len, int32_t has_divisor, float divisor,
                          b2s_boxavg **out);
void    b2s_boxavg_destroy(b2s_boxavg *p);
int32_t b2s_boxavg_reset(b2s_boxavg *p);
int32_t b2s_boxavg_exec(b2s_boxavg *p, const void *d_in, size_t n_in, void *d_out, size_t n_out_cap,
                        size_t max_calls, size_t *consumed, size_t *produced, size_t *calls, int32_t *call_again,
                        int32_t *done);

/* ---- the ADS-B receiver's PreambleDetector, Demodulator and Decoder::check_crc (≙ examples/adsb/src/
 * preamble_detector.rs:65-146, demodulator.rs:49-113, decoder.rs:57-73) as one block over three aligned f32 streams:
 * the samples |x|^2, the noise floor nf and the preamble correlation corr.  The detector's tags are not stream tags:
 * they are the detection list (index, correlation ratio), and each detection whose 480-sample window is complete is
 * demodulated into 112 PPM bits, CRC-checked and appended to the packet list (bytes MSB first).
 *   create: threshold must be finite and >= 0 (B2S_EINVAL otherwise); forward_failed_crc != 0 makes
 *           drain_packets return the frames that fail the CRC too (Decoder::new(true)).
 *   exec:   L = min(n_samples, n_nf, n_corr) (at most 2^30 per exec).  Scans the positions below L - 64 from where the
 *           last exec left off and consumes L - 544 (saturating) of every input: every detection below that already
 *           has its window.  With finished != 0 it is the last exec: the pending detections g with g + 480 < D (D =
 *           where the scan ended) are demodulated, the rest dropped, L is consumed and *done is set; later execs do
 *           nothing.  Stream-ordered, no synchronisation, except when the exec's worst case (one detection per 31
 *           positions) does not fit a list's capacity: the list then doubles, which synchronises.  The host bounds the
 *           lists by their true lengths once a copy of the counts behind an earlier exec has landed, so an undrained
 *           block grows its lists with what it detects, not with the positions it scans.  Slices need 4-byte alignment.
 *   drain_*: synchronise, copy up to cap entries in stream order to `host` (*n of them), and remove them.
 *   reset:  back to the stream's start, lists emptied. */
typedef struct {
    uint64_t preamble_index;       /* stream index of the preamble's start */
    float    preamble_correlation; /* the largest corr / nf of the trigger's window */
    int32_t  crc_passed;
    uint8_t  bytes[14];            /* the 112 bits, MSB first */
} b2s_adsb_packet;
typedef struct {
    uint64_t index;
    float    value;
} b2s_adsb_detection;
typedef struct b2s_adsb b2s_adsb;
int32_t b2s_adsb_create(b2s_ctx *ctx, float threshold, int32_t forward_failed_crc, b2s_adsb **out);
void    b2s_adsb_destroy(b2s_adsb *p);
int32_t b2s_adsb_reset(b2s_adsb *p);
int32_t b2s_adsb_exec(b2s_adsb *p, const float *d_samples, size_t n_samples, const float *d_nf, size_t n_nf,
                      const float *d_corr, size_t n_corr, int32_t finished, size_t *consumed, int32_t *done);
int32_t b2s_adsb_drain_packets(b2s_adsb *p, b2s_adsb_packet *host, size_t cap, size_t *n);
int32_t b2s_adsb_drain_detections(b2s_adsb *p, b2s_adsb_detection *host, size_t cap, size_t *n);

/* ---- Mueller & Muller clock recovery (≙ examples/zigbee/src/clock_recovery_mm.rs:28-97), f32 -> f32, bit for bit.
 *   create: omega, gain_omega, mu, gain_mu and omega_relative_limit must be finite, omega * omega_relative_limit must
 *           be >= 0 (f32::clamp panics otherwise) and look_ahead = ceil(omega + omega * omega_relative_limit + gain_mu)
 *           (f32, saturating cast) must be >= 1 (the loop reads i[ii + 1]); B2S_EINVAL otherwise.
 *   exec:   the reference's loop over one slice: while ii + look_ahead < n_in and oo < n_out_cap, one output per step.
 *           Consumption depends on the data, so the call SYNCHRONISES once to return *consumed (ii) and *produced (oo).
 *           A NaN latches mu: from then on nothing is consumed and every call fills its output.  A step that would
 *           move ii past n_in (|input| far above the loop's design range, or +inf) is B2S_ESTATE: *consumed /
 *           *produced and the block's state are those before that step.  Slices: 4-byte aligned, disjoint.
 *   reset:  back to the parameters given to create. */
typedef struct b2s_mmclock b2s_mmclock;
int32_t b2s_mmclock_create(b2s_ctx *ctx, float omega, float gain_omega, float mu, float gain_mu,
                           float omega_relative_limit, b2s_mmclock **out);
void    b2s_mmclock_destroy(b2s_mmclock *p);
int32_t b2s_mmclock_reset(b2s_mmclock *p);
size_t  b2s_mmclock_look_ahead(const b2s_mmclock *p);
int32_t b2s_mmclock_exec(b2s_mmclock *p, const float *d_in, size_t n_in, float *d_out, size_t n_out_cap,
                         size_t *consumed, size_t *produced);

/* ---- the ZigBee (IEEE 802.15.4 O-QPSK) chip decoder (≙ examples/zigbee/src/decoder.rs:78-183) with the Mac's FCS
 * check (mac.rs:62-85), one f32 stream input, frames out as a list.  Chip = v > 0; a 32-chip shift register matched
 * against the 16 chip sequences with mask 0x7FFFFFFE and Hamming distance < threshold.
 *   exec:   consumes the whole slice (4-byte aligned); stream-ordered, no synchronisation except when the exec's worst
 *           case (one frame per 192 chips) does not fit the list's capacity, which doubles it (see ADS-B above).
 *   drain:  synchronises, copies up to cap frames in stream order to `host` (*n of them) and removes them.
 *   reset:  back to the stream's start (Search, empty shift register), list emptied. */
typedef struct {
    uint64_t index;       /* stream index of the chip that completed the frame */
    uint32_t len;         /* bytes posted, FCS included (1..127) */
    int32_t  crc_ok;      /* Mac::calc_crc(bytes) == 0 && len > 2 */
    uint8_t  bytes[128];  /* bytes[0..len) */
} b2s_zigbee_frame;
typedef struct b2s_zigbee b2s_zigbee;
int32_t b2s_zigbee_create(b2s_ctx *ctx, uint32_t threshold, b2s_zigbee **out);
void    b2s_zigbee_destroy(b2s_zigbee *p);
int32_t b2s_zigbee_reset(b2s_zigbee *p);
int32_t b2s_zigbee_exec(b2s_zigbee *p, const float *d_in, size_t n_in, size_t *consumed);
int32_t b2s_zigbee_drain_frames(b2s_zigbee *p, b2s_zigbee_frame *host, size_t cap, size_t *n);

/* ---- the keyfob receiver's Decoder (≙ examples/keyfob/src/decoder.rs:64-127 with print, :36-52), one u8 stream
 * input, key codes out as a list.  An edge is a 1 while Down or a 0 while Up (other values are ignored); diff = its
 * position minus the last edge's.  diff in 63..=83 sets `output`, or, if it was set, clears it and appends a bit;
 * 131..=161 clears it and appends a bit (a rising edge appends 0, a falling edge 1); any other diff flushes the string
 * through print: a string holding 10101111 is reported from its first occurrence on.  A string still pending when the
 * input ends is never reported, as in the reference.
 *   exec:   consumes the whole slice (any alignment); stream-ordered, no synchronisation except when the exec's worst
 *           case (one code per 8 * 63 items, plus 2) does not fit the list's capacity, which doubles it.
 *   drain:  synchronises, copies up to cap codes in stream order to `host` (*n of them) and removes them.
 *   reset:  back to the stream's start (Down(0), output false, empty string), list emptied. */
#define B2S_KEYFOB_NONE  0
#define B2S_KEYFOB_CLOSE 1   /* the string ends in 11010101 */
#define B2S_KEYFOB_OPEN  2   /* 11100011 */
#define B2S_KEYFOB_TRUNK 3   /* 10111001 */
typedef struct {
    uint64_t index;       /* stream position of the flushing edge */
    uint32_t n_bits;      /* length after the prefix strip (>= 8; saturates at 2^32 - 1) */
    int32_t  label;       /* B2S_KEYFOB_*, from the string's true last 8 bits even when n_bits > 256 */
    uint8_t  bits[32];    /* the first min(n_bits, 256) bits, MSB first; the rest 0 */
} b2s_keyfob_code;
typedef struct b2s_keyfob b2s_keyfob;
int32_t b2s_keyfob_create(b2s_ctx *ctx, b2s_keyfob **out);
void    b2s_keyfob_destroy(b2s_keyfob *p);
int32_t b2s_keyfob_reset(b2s_keyfob *p);
int32_t b2s_keyfob_exec(b2s_keyfob *p, const uint8_t *d_in, size_t n_in, size_t *consumed);
int32_t b2s_keyfob_drain_codes(b2s_keyfob *p, b2s_keyfob_code *host, size_t cap, size_t *n);

/* ---- tap design, host side, f64 then cast (≙ futuredsp::firdes::kaiser, firdes/basic.rs:310-459)
 * Return the tap count; write taps only if cap is large enough (call with taps=NULL to size). */
size_t b2s_firdes_kaiser_lowpass(double cutoff, double transition_bw, double max_ripple,
                                 float *taps, size_t cap);
size_t b2s_firdes_kaiser_multirate(size_t interp, size_t decim, size_t half_polyphase_len,
                                   double max_ripple, float *taps, size_t cap);
/* ≙ futuredsp::windows::hamming (windows.rs:68-120, gen_cos with {0.54, 0.46}): len f64 points, periodic != 0 computes
 * len + 1 and drops the last.  Same count / cap convention; len == 0 returns 0. */
size_t b2s_window_hamming(size_t len, int32_t periodic, double *out, size_t cap);
/* ≙ futuredsp::firdes::hilbert (firdes/basic.rs:202-222): taps of the window's length, f64 then cast to f32.
 * The reference asserts an odd length: an even (or zero) length returns 0 taps. */
size_t b2s_firdes_hilbert(const double *window, size_t len, float *taps, size_t cap);
/* ≙ futuredsp::firdes::lowpass (firdes/basic.rs:25-42): the windowed sinc, one tap per window entry, f64 then cast to
 * f32.  The reference asserts |cutoff| < 1/2: a cutoff outside that (or NaN), or len == 0, returns 0 taps. */
size_t b2s_firdes_lowpass(double cutoff, const double *window, size_t len, float *taps, size_t cap);

/* ---- the LoRa transmitter (≙ examples/lora/src/encoder.rs:33-284, modulator.rs:46-152, transmitter.rs:34-168 with
 * build_upchirp_phase_coherent and samples_from_phase_diff, utils.rs:917-963).  Configuration as Encoder::new: sf 5..12,
 * code_rate 1..4 (CR 4/5 .. 4/8), has_crc, ldro_enabled, implicit_header (B2S_EINVAL otherwise).  A payload of more than
 * B2S_LORA_MAX_PAYLOAD bytes, or of fewer than 2 bytes with has_crc, is B2S_EINVAL (the reference panics on both) and
 * then nothing of the call is encoded or queued.  An empty payload without CRC is a frame of one interleaver block.
 *   symbol_count: the u16 symbols Encoder::encode makes of a payload of payload_len bytes (host only).
 *   encode:       a batch on the device: frame i is lengths[i] (HOST array) bytes of d_payloads, back to back, and its
 *                 symbols follow those of frame i - 1 in d_symbols; *n_symbols is their total.  symbols_cap below
 *                 the total is B2S_EINVAL.  Asynchronous on the context's stream. */
#define B2S_LORA_MAX_PAYLOAD 255
int32_t b2s_lora_symbol_count(int32_t sf, int32_t code_rate, int32_t has_crc, int32_t ldro_enabled,
                              int32_t implicit_header, size_t payload_len, size_t *n_symbols);
int32_t b2s_lora_encode(b2s_ctx *ctx, int32_t sf, int32_t code_rate, int32_t has_crc, int32_t ldro_enabled,
                        int32_t implicit_header, const uint8_t *d_payloads, const size_t *lengths, size_t n_frames,
                        uint16_t *d_symbols, size_t symbols_cap, size_t *n_symbols);
/* Transmitter: a source of Complex<f32> samples, the concatenation of its frames, bit-identical to the reference under
 * any slicing of the stream (cos / sin: see DESIGN §4.19).  A frame of n_sym symbols has
 * 2 pad + (preamble_len + 4 [+ 2 if sf < 7]) N + N/4 - OS + n_sym N samples, N = 2^sf OS.
 *   create:        sync_symbols is the expanded sync word (SynchWord::verify_and_expand); a symbol >= 2^sf,
 *                  oversampling == 0, 2^sf oversampling > 2^20, or a frame that could exceed 2^32 - 1 samples is
 *                  B2S_EINVAL.
 *   push:          the `msg` handler for n_frames payloads (HOST memory, back to back): queues them in order and
 *                  encodes them on the device.  May wait for the context's stream when a device buffer grows.
 *   set_sync_word: the `synch_word` handler; applies to every frame whose first sample has not been produced yet.
 *                  A refused word (B2S_EINVAL) leaves the old one in place.
 *   exec:          writes the next min(n_out_cap, pending) samples of the stream to d_out (8-byte aligned); one exec
 *                  may span several frames.  Stream-ordered, never synchronises.  *finished is set once finish has been
 *                  called and every queued sample has been produced (Pmt::Finished, transmitter.rs:79, :134-136).
 *   drain_bursts:  the burst_start tags (transmitter.rs:129-132, :153-159) of the frames whose first sample has been
 *                  produced, in stream order, up to cap of them (*n); they are removed.
 *   reset:         drops the queue, the stream position, the bursts and the finish; the sync word returns to create's. */
typedef struct {
    uint64_t index;       /* stream index of the frame's first sample */
    uint64_t len;         /* the frame's samples */
} b2s_lora_burst;
typedef struct b2s_lora_tx b2s_lora_tx;
int32_t b2s_lora_tx_create(b2s_ctx *ctx, int32_t sf, int32_t code_rate, int32_t has_crc, int32_t ldro_enabled,
                           int32_t implicit_header, size_t oversampling, const uint32_t sync_symbols[2],
                           size_t preamble_len, size_t pad, b2s_lora_tx **out);
void    b2s_lora_tx_destroy(b2s_lora_tx *p);
int32_t b2s_lora_tx_reset(b2s_lora_tx *p);
int32_t b2s_lora_tx_push(b2s_lora_tx *p, const uint8_t *payloads, const size_t *lengths, size_t n_frames);
int32_t b2s_lora_tx_set_sync_word(b2s_lora_tx *p, uint32_t sync0, uint32_t sync1);
int32_t b2s_lora_tx_finish(b2s_lora_tx *p);
int32_t b2s_lora_tx_pending(const b2s_lora_tx *p, uint64_t *samples);   /* queued samples not yet produced */
int32_t b2s_lora_tx_exec(b2s_lora_tx *p, void *d_out, size_t n_out_cap, size_t *produced, int32_t *finished);
int32_t b2s_lora_tx_drain_bursts(b2s_lora_tx *p, b2s_lora_burst *host, size_t cap, size_t *n);

/* ---- the WLAN transmitter (≙ examples/wlan/src/mac.rs:16-103, encoder.rs:22-277, mapper.rs:23-132, the
 * Fft::with_options(64, Inverse, true, sqrt(1/52)) of bin/tx.rs:53-59 and prefix.rs:57-141).  MCS numbers follow the
 * reference's Mcs enum (B2S_WLAN_*); a payload is the MAC data frame's body, at most B2S_WLAN_MAX_PAYLOAD bytes, and
 * its PSDU adds the 24-byte header and the 4-byte FCS.  One OFDM symbol is 48 subcarrier bytes (split_symbols: n_bpsc
 * coded bits each), and a frame is its SIGNAL symbol followed by FrameParam::n_symbols data symbols.
 *   frame_param: FrameParam::new (lib.rs:323-363) of a PSDU of psdu_len bytes (at most B2S_WLAN_MAX_PSDU).
 *   encode:      Mac + Encoder + the SIGNAL field over a batch, from a fresh encoder (zero bit buffer) whose scrambler
 *                seed (1..127) and sequence number (0..4095) are given: frame i is lengths[i] bytes of d_payloads
 *                (device, back to back) at MCS mcs[i] (HOST arrays).  Each frame writes 48 (1 + n_symbols) bytes to
 *                d_symbols, frame after frame; *n_symbols is the OFDM symbol total.  symbols_cap below it, or an
 *                oversized payload, is B2S_EINVAL and nothing is encoded.  Asynchronous on the context's stream.
 * Pad bits are the reference's: encoder.rs never clears its bit buffer, so the pad bits of a frame are the bits an
 * earlier, longer frame left there (DESIGN §4.20). */
#define B2S_WLAN_BPSK_1_2   0
#define B2S_WLAN_BPSK_3_4   1
#define B2S_WLAN_QPSK_1_2   2
#define B2S_WLAN_QPSK_3_4   3
#define B2S_WLAN_QAM16_1_2  4
#define B2S_WLAN_QAM16_3_4  5
#define B2S_WLAN_QAM64_2_3  6
#define B2S_WLAN_QAM64_3_4  7
#define B2S_WLAN_MAX_PAYLOAD 1500
#define B2S_WLAN_MAX_PSDU    1528
int32_t b2s_wlan_frame_param(int32_t mcs, size_t psdu_len, size_t *n_symbols, size_t *n_data_bits, size_t *n_pad);
int32_t b2s_wlan_encode(b2s_ctx *ctx, const uint8_t src[6], const uint8_t dst[6], const uint8_t bss[6],
                        uint32_t sequence_number, uint32_t scrambler_seed, const uint8_t *d_payloads,
                        const size_t *lengths, const int32_t *mcs, size_t n_frames, uint8_t *d_symbols,
                        size_t symbols_cap, size_t *n_symbols);
/* Transmitter: a source of Complex<f32> samples, the concatenation of the Prefix block's bursts.  A frame of n OFDM
 * symbols (SIGNAL included) has pad_front + 320 + 80 n + max(pad_tail, 1) samples.  The FFT is the library's own
 * 64-point inverse transform (bit-identical to b2s_fft_* with shift and norm sqrtf(1/52)), so the samples are not the
 * reference's bits (rustfft's); everything around it is its f32 arithmetic in its order.  The sample after the last
 * symbol is windowed against 0 (the reference reads a buffer slot it has not written there).
 *   create:       the Mac's three addresses and the Encoder's default MCS; pads above 2^32 - 1 are B2S_EINVAL.
 *   push:         the Mac's `tx` handler for n_frames payloads (HOST memory, back to back): mcs NULL, or mcs[i] == -1,
 *                 is the default MCS (Pmt::Blob), otherwise frame i's (the (data, mcs) pair).  A payload above
 *                 B2S_WLAN_MAX_PAYLOAD or an MCS outside -1..7 is B2S_EINVAL and nothing is queued.  Frames are never
 *                 dropped (the reference's encoder queue holds 1000).  Sequence number and scrambler seed advance per
 *                 frame.  May wait for the context's stream when a device buffer grows.
 *   exec:         writes the next min(n_out_cap, pending) samples to d_out (8-byte aligned); one exec may span
 *                 several frames.  Stream-ordered, never synchronises.  *finished is set once finish has been called
 *                 and every queued sample has been produced.
 *   drain_bursts: the burst_start tags (prefix.rs:133) of the frames whose first sample has been produced, in stream
 *                 order, up to cap of them (*n); they are removed.
 *   reset:        the created state: seed 1, sequence number 0, a zero bit buffer, no queue, position 0, no finish. */
typedef struct {
    uint64_t index;       /* stream index of the frame's first sample */
    uint64_t len;         /* the frame's samples */
} b2s_wlan_burst;
typedef struct b2s_wlan_tx b2s_wlan_tx;
int32_t b2s_wlan_tx_create(b2s_ctx *ctx, const uint8_t src[6], const uint8_t dst[6], const uint8_t bss[6],
                           int32_t default_mcs, size_t pad_front, size_t pad_tail, b2s_wlan_tx **out);
void    b2s_wlan_tx_destroy(b2s_wlan_tx *p);
int32_t b2s_wlan_tx_reset(b2s_wlan_tx *p);
int32_t b2s_wlan_tx_push(b2s_wlan_tx *p, const uint8_t *payloads, const size_t *lengths, const int32_t *mcs,
                         size_t n_frames);
int32_t b2s_wlan_tx_finish(b2s_wlan_tx *p);
int32_t b2s_wlan_tx_pending(const b2s_wlan_tx *p, uint64_t *samples);   /* queued samples not yet produced */
int32_t b2s_wlan_tx_exec(b2s_wlan_tx *p, void *d_out, size_t n_out_cap, size_t *produced, int32_t *finished);
int32_t b2s_wlan_tx_drain_bursts(b2s_wlan_tx *p, b2s_wlan_burst *host, size_t cap, size_t *n);

/* ---- the ZigBee transmitter (≙ examples/zigbee/src/mac.rs:135-252, modulator.rs:4-342 and iq_delay.rs:11-139: the
 * Mac -> modulator -> IqDelay chain of bin/tx.rs:37-56).  A payload of n bytes (at most B2S_ZIGBEE_MAX_PAYLOAD)
 * becomes the Mac's frame of n + 16 bytes: 00 00 00 a7, n + 11, 41 88, the sequence number, aa 1a ff ff 44 33, the
 * payload and the FCS (calc_crc over bytes 5 .. 14 + n, little endian).  The modulator makes 128 samples of each byte
 * (16 DSSS chips per nibble, low nibble first, each chip 4 samples of SHAPE, in f32); IqDelay delays Q by two
 * samples and pads each frame with pad zeros before and after it.  A frame has 2 pad + 128 (n + 16) + 2 samples.
 * There is no FEC: push frames the payloads on the host and copies their bytes to the device.
 * Transmitter: a source of Complex<f32> samples, the concatenation of IqDelay's frames, bit-identical to the reference
 * (the sign of every zero included) under any slicing of the stream.
 *   create:       pad is IqDelay's PADDING (B2S_ZIGBEE_PADDING in the reference); above 2^32 - 1 is B2S_EINVAL.
 *   push:         the Mac's `tx` handler for n_frames payloads (HOST memory, back to back).  A payload above
 *                 B2S_ZIGBEE_MAX_PAYLOAD is dropped on its own, as the Mac drops it, and the others are queued in order;
 *                 *n_dropped counts the dropped ones.  The sequence number (a u8) advances per queued frame only.  Frames
 *                 are never dropped for queue length (the Mac's 128-frame bound depends on its scheduler).  May wait
 *                 for the context's stream when a device buffer grows.
 *   exec:         writes the next min(n_out_cap, pending) samples to d_out (8-byte aligned); one exec may span several
 *                 frames.  Stream-ordered, never synchronises.  *finished is set once finish has been called and every
 *                 queued sample has been produced, the last frame's tail pad included (the reference's graph never
 *                 finishes).
 *   drain_bursts: the burst_start tags (iq_delay.rs:112-118) of the frames whose first sample has been produced, in
 *                 stream order, up to cap of them (*n); they are removed.  A tag sits on the frame's first front-pad
 *                 sample and its value is the frame's length.
 *   reset:        the created state: sequence number 0, no queue, position 0, no finish. */
#define B2S_ZIGBEE_MAX_PAYLOAD 116
#define B2S_ZIGBEE_PADDING     40000
typedef struct {
    uint64_t index;       /* stream index of the frame's first sample */
    uint64_t len;         /* the frame's samples */
} b2s_zigbee_burst;
typedef struct b2s_zigbee_tx b2s_zigbee_tx;
int32_t b2s_zigbee_tx_create(b2s_ctx *ctx, size_t pad, b2s_zigbee_tx **out);
void    b2s_zigbee_tx_destroy(b2s_zigbee_tx *p);
int32_t b2s_zigbee_tx_reset(b2s_zigbee_tx *p);
int32_t b2s_zigbee_tx_push(b2s_zigbee_tx *p, const uint8_t *payloads, const size_t *lengths, size_t n_frames,
                           size_t *n_dropped);
int32_t b2s_zigbee_tx_finish(b2s_zigbee_tx *p);
int32_t b2s_zigbee_tx_pending(const b2s_zigbee_tx *p, uint64_t *samples);   /* queued samples not yet produced */
int32_t b2s_zigbee_tx_exec(b2s_zigbee_tx *p, void *d_out, size_t n_out_cap, size_t *produced, int32_t *finished);
int32_t b2s_zigbee_tx_drain_bursts(b2s_zigbee_tx *p, b2s_zigbee_burst *host, size_t cap, size_t *n);

#ifdef __cplusplus
}
#endif
#endif /* B200SDR_H */
