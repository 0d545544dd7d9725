/*
 * llama2_oracle.h — CPU parity oracle for the llama2.zig decode hot path.
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / `--impl reference` legs may load this library.  The
 * product (libllama2_b200.so) never links, loads or calls anything in oracle/.
 *
 * What it is: a plain-C restatement of src/main.zig:285-713
 * (transformer() and the numeric helpers it calls) that keeps the reference's
 * exact SIMD lane / accumulator summation order, parameterised by the vector
 * width W = DEFAULT_VECTOR_WIDTH (src/main.zig:7; 4, 8 or 16 depending on the
 * host the Zig compiler targets; default 8 = AVX2, the README machine).
 *
 * Pinning status (read before trusting it):
 *   - PINNED by the reference's own unit tests, re-expressed in
 *     tests/test_oracle_kats.py: `matrix_multiplies` (src/main.zig:1078-1087),
 *     `vector_length_less_than_width_case` (:1089-1103),
 *     `vector_weighted_sum_rows` (:1117-1139), `softmax` (:1141-1150).
 *   - END-TO-END transformer() PARITY IS UNPINNED BY THE REFERENCE: the
 *     reference has no test that calls transformer(), ships no golden logits or
 *     text, and there is no Zig toolchain in this image, so the Zig binary cannot
 *     be run to make one.  The 221-token stories15M stream in
 *     tests/golden/stories15M_t0_tokens.json is *derived* (SURVEY.md Appendix B:
 *     it is invariant under W in {4,8,16}, ordered vs tree lane reduction, and
 *     fp64), not produced by the Zig binary.
 *   - Transcendentals: Zig's std.math.exp/cos/sin/pow are Zig's own software
 *     routines; this oracle uses glibc expf/cosf/sinf/powf, which may differ in
 *     the last ulp.  That is inside the north-star tolerance (logits 1e-4 rel).
 *
 * Float mode: src/main.zig:11-13 requests @setFloatMode(.optimized) in a
 * container-level comptime block; whether it reaches the functions cannot be
 * settled without a Zig compiler.  Two builds of this file exist:
 *   liborc_strict.so  -O2 -ffp-contract=off, @reduce(.Add) as an ORDERED lane
 *                     reduction — the parity oracle;
 *   liborc_fast.so    -O3 -mfma -ffp-contract=fast -DORC_OPTIMIZED=1, tree lane
 *                     reduction — the CPU speed baseline and a sensitivity check.
 */
#ifndef LLAMA2_ORACLE_H
#define LLAMA2_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ConfigReader, src/main.zig:17-25 (vocab_size already abs(); see :942-944). */
typedef struct orc_config {
    int32_t dim, hidden_dim, n_layers, n_heads, n_kv_heads, vocab_size, seq_len;
} orc_config;

typedef struct orc_model orc_model;

/* ---- primitive ops (each cites the function it restates) ------------------ */
/* matmul, src/main.zig:485-498 -> matmul_fused(N=1), 8 accumulators (:546).   */
void  orc_matmul(float *xout, const float *x, const float *w, int d, int n, int W);
/* matmul_fused(N=2|3), src/main.zig:530-605, 4 accumulators (:546).           */
void  orc_matmul_fused2(float *o0, float *o1, const float *x, const float *w0,
                        const float *w1, int d, int n, int W);
void  orc_matmul_fused3(float *o0, float *o1, float *o2, const float *x, const float *w0,
                        const float *w1, const float *w2, int d, int n, int W);
/* rmsnorm, src/main.zig:432-468 (o may alias x, :426).                         */
void  orc_rmsnorm(float *o, const float *x, const float *w, int n, int W);
/* vector_dot_product, src/main.zig:503-527.                                    */
float orc_dot(const float *x, const float *y, int n, int W);
/* vector_mul, src/main.zig:608-628.                                            */
void  orc_vector_mul(float *x, const float *y, int n, int W);
/* vector_weighted_sum_rows, src/main.zig:657-685.                              */
void  orc_weighted_sum_rows(float *xout, int out_len, const float *rows, int row_stride,
                            const float *weights, int n_weights, int W);
/* softmax, src/main.zig:687-706 (scalar, sequential).                          */
void  orc_softmax(float *x, int n);
/* accum, src/main.zig:708-713.                                                 */
void  orc_accum(float *a, const float *b, int n);
/* argmax, src/main.zig:715-726 (first maximum wins: strict '>').               */
int   orc_argmax(const float *x, int n);
/* RoPE angle for pair index i (even) at position pos, src/main.zig:338-342.    */
void  orc_rope_angle(int i, int head_size, int pos, float *fcr, float *fci);

/* ---- model: Weights.init (src/main.zig:73-115) + RunState.init (:137-154) -- */
/* `data` = the checkpoint after the 28-byte header (src/main.zig:955-967);
 * BORROWED for the life of the model.  W in {4,8,16}.                          */
orc_model *orc_model_create(const orc_config *cfg, const float *data, int shared_weights, int W);
void       orc_model_destroy(orc_model *m);
/* transformer(), src/main.zig:285-430.  Writes logits (vocab_size floats).     */
void       orc_transformer(orc_model *m, int token, int pos);
float     *orc_logits(orc_model *m);
/* RunState views for layer-level parity checks: 0=x 1=xb 2=xb2 3=hb 4=hb2 5=q
 * 6=k 7=v 8=att 9=key_cache 10=value_cache.  Returns pointer, *len = floats.   */
float     *orc_state(orc_model *m, int which, uint64_t *len);
/* Number of floats a checkpoint of this config holds after the header
 * (src/main.zig:85-112).                                                       */
uint64_t   orc_checkpoint_floats(const orc_config *cfg, int shared_weights);

/* Generation loop twin of src/main.zig:995-1042 at temperature 0 (argmax) with
 * optional teacher forcing.  forced[p] (if non-NULL) replaces the argmax as the
 * next token at position p (like prompt forcing, :999-1000).  stop_on_bos: break
 * when next == 1 (:1017-1019).  out_next[p] receives the token chosen at p.
 * Returns the number of transformer() calls.  *secs_after_first is the wall time
 * from after the first step to the end (the reference's timer convention,
 * :1038-1047).                                                                 */
int orc_generate(orc_model *m, int token0, int n_steps, const int32_t *forced,
                 int stop_on_bos, int32_t *out_next, double *secs_after_first);

/* ---- checkpoint file (legacy llama2.c layout) ------------------------------ */
/* Reads the 28-byte header (src/main.zig:936-946). Returns 0 on success.       */
int orc_read_header(const char *path, orc_config *cfg, int *shared_weights, uint64_t *file_floats);
/* Reads the float payload into dst (n floats). Returns 0 on success.           */
int orc_read_payload(const char *path, float *dst, uint64_t n);

/* ---- synthetic checkpoints (SURVEY.md 8d) ---------------------------------- */
/* Counter-based generator, bit-identical on CPU and GPU (integer hash + one
 * double multiply-add, no transcendentals).  Element i of a tensor:
 *   h = mix64(tensor_seed + (i+1)*0x9E3779B97F4A7C15)
 *   s = sum of the four 16-bit fields of h - 131070          (Irwin-Hall, n=4)
 *   v = (float)( (double)s * scale + mean ),  clipped to [lo, hi]
 * with scale = sigma / 37837.22723720648.                                      */
void orc_synth_fill(float *dst, uint64_t first, uint64_t count, uint64_t tensor_seed,
                    double mean, double sigma, float lo, float hi);
/* Fills a whole checkpoint payload (layout src/main.zig:85-112) with the
 * per-tensor distributions of SURVEY.md 8d.  data must hold
 * orc_checkpoint_floats() floats.                                              */
void orc_synth_checkpoint(const orc_config *cfg, int shared_weights, uint64_t seed, float *data);

#ifdef __cplusplus
}
#endif
#endif
