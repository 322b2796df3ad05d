/*
 * iir_oracle.c -- CPU restatement of futuredsp::IirFilter (crates/futuredsp/src/iir.rs:78-178).  TEST
 * INFRASTRUCTURE ONLY: loaded by tests/iir_oracle.py; the product (futuresdr_b200/ + libb200sdr.so) never links it.
 *
 * Every operation is the reference's, in its order, in the sample type: compile with -ffp-contract=off so the
 * compiler does not fuse a*b+c, which stable Rust never does.  Pinned by the reference's own vectors
 * (tests/golden/reference_iir_known_answers.json, replayed by tests/test_oracle_iir.py).
 */
#include <stddef.h>

/* futuredsp::ComputationStatus, crates/futuredsp/src/lib.rs:33-45 */
enum { ORC_INSUFFICIENT_INPUT = 0, ORC_INSUFFICIENT_OUTPUT = 1, ORC_BOTH_SUFFICIENT = 2 };


/* ------------------------------------------------------------------------------------------
 * IirFilter -- crates/futuredsp/src/iir.rs:78-178 (taps_accessor_work), one StatefulFilter::filter call.
 * state: memory[n_a] and its fill count *mem_len (in/out; Vec::len of the reference's memory).
 *   fill:   memory.push(i[memory.len()]) until n_a items; the call that fills returns (0, 0)     (:102-129)
 *   output: o = 0; o += b[j] * i[k + n_b - 1 - j]; o += a[j] * memory[j]; shift; memory[0] = o (:136-164)
 *   status: :166-177.  n_b == 0 is the reference's assert (:132): returns -1.
 * ---------------------------------------------------------------------------------------- */
#define ORC_IIR_WORK(NAME, T)                                                                                    \
int NAME(const T *a, size_t n_a, const T *b, size_t n_b, T *memory, size_t *mem_len, const T *in, size_t n_in,   \
         T *out, size_t n_out_cap, size_t *consumed, size_t *produced) {                                         \
    const int st_empty = n_out_cap == 0 ? ORC_BOTH_SUFFICIENT : ORC_INSUFFICIENT_INPUT;                         \
    *consumed = 0; *produced = 0;                                                                                \
    if (n_in == 0) return st_empty;                                                                              \
    size_t num_filled = 0;                                                                                       \
    while (*mem_len < n_a) {                                                                                     \
        if (n_in <= *mem_len) return st_empty;                                                                   \
        memory[*mem_len] = in[*mem_len];                                                                         \
        *mem_len += 1; num_filled++;                                                                             \
    }                                                                                                            \
    if (num_filled == n_in) return st_empty;                                                                     \
    if (n_b == 0) return -1;                                                                                     \
    size_t c = 0, p = 0;                                                                                         \
    while (c + n_b - 1 < n_in && p < n_out_cap) {                                                                \
        T o = 0;                                                                                                 \
        for (size_t j = 0; j < n_b; j++) o += b[j] * in[c + n_b - j - 1];                                        \
        for (size_t j = 0; j < n_a; j++) o += a[j] * memory[j];                                                  \
        for (size_t j = n_a; j-- > 1;) memory[j] = memory[j - 1];                                                \
        if (n_a) memory[0] = o;                                                                                  \
        out[p] = o;                                                                                              \
        p++; c++;                                                                                                \
    }                                                                                                            \
    *consumed = c; *produced = p;                                                                                \
    if (c == n_in && p == n_out_cap) return ORC_BOTH_SUFFICIENT;                                                 \
    if (c < n_in) return ORC_INSUFFICIENT_OUTPUT;                                                                \
    return ORC_INSUFFICIENT_INPUT;                                                                               \
}
ORC_IIR_WORK(orc_iir_work_f32, float)
ORC_IIR_WORK(orc_iir_work_f64, double)

/* f64 evaluation of an f32 filter over a whole stream (arbiter, not a reference function): the same recurrence and
 * memory fill with every value widened to double; n_out = n_in - n_b + 1 outputs. */
void orc_iir_exact_f32(const float *a, size_t n_a, const float *b, size_t n_b, const float *in, size_t n_in,
                       double *out) {
    double mem[64] = {0};
    if (n_a > 64 || n_b == 0 || n_in < n_a || n_in + 1 < n_b) return;
    for (size_t j = 0; j < n_a; j++) mem[j] = in[j];
    for (size_t k = 0; k + n_b - 1 < n_in; k++) {
        double o = 0;
        for (size_t j = 0; j < n_b; j++) o += (double)b[j] * (double)in[k + n_b - j - 1];
        for (size_t j = 0; j < n_a; j++) o += (double)a[j] * mem[j];
        for (size_t j = n_a; j-- > 1;) mem[j] = mem[j - 1];
        if (n_a) mem[0] = o;
        out[k] = o;
    }
}
