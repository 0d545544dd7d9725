/*
 * llama2_host.h — C++ twin of the reference's Zig host (everything in src/main.zig that is
 * NOT the hot path), written because no Zig toolchain exists in this image.  It drives the
 * C ABI of include/llama2_b200.h exactly where the patched Zig host would (INTEGRATION.md):
 *   checkpoint load      src/main.zig:936-967      -> l2h_load_checkpoint
 *   transformer() call   src/main.zig:996          -> l2b_forward(ctx, token, pos, logits)
 *   sampler              src/main.zig:715-798      -> l2h_argmax / l2h_sample / l2h_sample_top_p
 *   tokenizer            src/main.zig:166-283      -> l2h_tokenizer_*
 *   generation loop      src/main.zig:995-1050     -> l2h_generate
 * A small C surface is exported so bench.py can time the end-to-end loop (host buffers,
 * H2D/D2H inside the timed region) without Python in the way.
 */
#ifndef LLAMA2_HOST_H
#define LLAMA2_HOST_H

#include <stdint.h>

#include "../../include/llama2_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct l2h_checkpoint {
    l2b_config config;      /* vocab_size already abs(); shared_weights from its sign (:943) */
    float *data;            /* payload after the 28-byte header (:955-964), malloc'ed        */
    uint64_t n_floats;
} l2h_checkpoint;

int32_t l2h_load_checkpoint(const char *path, l2h_checkpoint *out);
void l2h_free_checkpoint(l2h_checkpoint *ck);

typedef struct l2h_tokenizer l2h_tokenizer;
int32_t l2h_tokenizer_load(const char *path, int32_t vocab_size, l2h_tokenizer **out);   /* :173-196 */
void l2h_tokenizer_free(l2h_tokenizer *t);
int32_t l2h_tokenizer_max_token_len(const l2h_tokenizer *t);
const char *l2h_tokenizer_token(const l2h_tokenizer *t, int32_t id, int32_t *len);
int32_t l2h_tokenizer_lookup(const l2h_tokenizer *t, const char *bytes, int32_t len);     /* :208-215, -1 = none */
/* encode (:219-282): returns number of tokens written (<= cap), or a negative error        */
int32_t l2h_tokenizer_encode(const l2h_tokenizer *t, const char *text, int32_t len, int32_t *out, int32_t cap);

int32_t l2h_argmax(const float *x, int32_t n);                                             /* :715-726 */
void l2h_softmax(float *x, int32_t n);                                                     /* :687-706 (sampler use, :1008) */
void l2h_seed(uint64_t seed);                                                              /* :845, :926 */
int32_t l2h_sample(const float *probs, int32_t n);                                         /* :728-741 */
int32_t l2h_sample_top_p(const float *probs, int32_t n, float p, void *scratch_2n_words);  /* :754-798 */
/* :770-797 on a candidate list that already passed the cutoff of :761-768 (sorted here)      */
int32_t l2h_sample_top_p_candidates(l2b_prob_index *cand, int32_t n_cand, float p);
/* The same three with the uniform draw ("coin", in [0, 1)) passed in: each of the above draws one coin
 * from the PRNG and calls its _r form, except that l2h_sample_top_p draws nothing (and returns the argmax)
 * when no entry passes the cutoff; l2h_sample_top_p_r then does not read the coin either.              */
int32_t l2h_sample_r(const float *probs, int32_t n, float coin);
int32_t l2h_sample_top_p_r(const float *probs, int32_t n, float p, void *scratch_2n_words, float coin);
int32_t l2h_sample_top_p_candidates_r(l2b_prob_index *cand, int32_t n_cand, float p, float coin);
/* Prints token `next` as the reference does after `token` (:1022-1034).                       */
void l2h_print_token(const l2h_tokenizer *t, int32_t token, int32_t next);

typedef struct l2h_gen_options {
    float temperature;      /* :840, 0 => argmax                                             */
    float top_p;            /* :841                                                          */
    int32_t n_steps;        /* :842, :992-993                                                */
    int32_t stop_on_bos;    /* :1017-1019 (1 in the reference)                               */
    int32_t use_device_argmax; /* 0: l2b_forward + host sampler (reference data flow);
                                  1: l2b_forward_argmax (only the token id crosses PCIe)      */
    int32_t use_prefill;       /* 1: the prompt positions go through l2b_prefill (no logits, no
                                  host round trip per prompt token; :996-1000)                */
    int32_t use_device_sampler;/* 1, temperature > 0: l2b_forward_sample does logits/=T, softmax and
                                  the top-p prefilter on the GPU (:1005-1008, :761-768); the host
                                  only sorts the candidates and draws (:770-797)               */
} l2h_gen_options;

typedef struct l2h_gen_result {
    int32_t n_forward;          /* transformer() calls made                                  */
    int32_t n_tokens;           /* tokens written to out_tokens                              */
    double secs_total;          /* whole loop                                                */
    double secs_after_first;    /* the reference's timer: starts after the first token (:1038-1047) */
    uint64_t h2d_bytes, d2h_bytes;  /* bytes moved across PCIe by the loop                   */
} l2h_gen_result;

/* The generation loop of src/main.zig:995-1042 over the C ABI.  prompt/n_prompt: forced
 * tokens (:999-1000).  out_tokens receives `next` per step (cap entries).  If print_tok is
 * non-NULL tokens are detokenised to stdout as the reference does (:1022-1034).             */
int32_t l2h_generate(l2b_ctx *ctx, const l2b_config *cfg, const l2h_gen_options *opt,
                     const int32_t *prompt, int32_t n_prompt, const l2h_tokenizer *print_tok,
                     int32_t *out_tokens, int32_t cap, l2h_gen_result *res);

/* Sampled speculative decoding: the device-sampler loop of l2h_generate (l2b_forward_sample on the target,
 * then l2h_sample / l2h_sample_top_p_candidates / l2h_sample_top_p with the PRNG of l2h_seed) from `token` at
 * `pos`, a round at a time.  Each round the draft (another context or session with the same vocabulary and a
 * seq_len at least the target's) proposes kk = min(k, tokens still wanted - 1, seq_len - 1 - p) tokens, each
 * one l2b_forward_sample and the _r sampler with the coin the target would use for that token if every
 * earlier proposal is accepted (peeked, not drawn).  One l2b_verify_sample_ragged then gives the target's
 * sampler output at every position of [t, d_1 .. d_kk]; the host walks them with the same sampler, consuming
 * coins exactly as the plain loop does, and emits tokens up to the first that differs from the next draft (or
 * BOS, with stop_on_bos).  Coins peeked and not consumed stay queued for the tokens they belong to.  So
 * out_next[0 .. *n_done), *n_done and the target's KV rows [0, pos + *n_done) are those of the plain loop with
 * the same seed, bit for bit, whatever the draft, and the PRNG is left where that loop leaves it.  Afterwards
 * target and draft both hold the stream's rows [0, pos + *n_done) (rows past it are stale), so a second call
 * from (out_next[*n_done - 1], pos + *n_done) continues the stream.  *n_rounds (n_rounds may be NULL) counts
 * rounds.  cfg and draft_cfg are the two models' configs.  NULL pointers, target == draft, k outside [0,
 * L2B_SPECULATIVE_MAX_K], n_steps < 0, temperature not > 0 (greedy: l2b_generate_speculative), top_p outside
 * [0, 1], another vocab_size, a smaller draft seq_len, or token / pos out of range => L2B_ERR_INVALID_ARG
 * before anything runs; a library error is returned as is (see l2b_last_error of target or draft).       */
int32_t l2h_generate_speculative_sample(l2b_ctx *target, const l2b_config *cfg, l2b_ctx *draft,
                                        const l2b_config *draft_cfg, int32_t token, int32_t pos, int32_t n_steps,
                                        int32_t k, float temperature, float top_p, int32_t stop_on_bos,
                                        int32_t *out_next, int32_t *n_done, int32_t *n_rounds);

#ifdef __cplusplus
}
#endif
#endif
