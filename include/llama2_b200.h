/*
 * llama2_b200.h — C ABI of the H100 (sm_90a) decode hot path for cgbur/llama2.zig.
 *
 * This library replaces ONE internal call of the reference,
 *     transformer(token, pos, &config, &state, &weights)      src/main.zig:285, call site :996
 * and the numeric helpers it calls (src/main.zig:432-713).  The reference has no FFI of
 * its own; these entry points are what its Zig host declares `extern "c"` (see
 * INTEGRATION.md for the patch).  Everything else (CLI, checkpoint and tokenizer
 * loaders, sampler) stays in the host.
 *
 * Conventions
 *   - plain C types only; every call returns L2B_OK (0) or a negative l2b_status and never
 *     aborts or throws across the boundary (the reference's `assert`s, e.g. :433-434,
 *     :534-540, become argument checks);
 *   - host pointers are borrowed for the duration of the call only;
 *   - one context = one decode stream on 1, 2, 4 or 8 GPUs; not thread-safe (the reference is
 *     single-threaded);
 *   - there is NO CPU fallback: if no sm_90 device is usable the call fails with
 *     L2B_ERR_CUDA / L2B_ERR_NO_DEVICE.
 */
#ifndef LLAMA2_B200_H
#define LLAMA2_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define L2B_ABI_VERSION 2

typedef enum l2b_status {
    L2B_OK = 0,
    L2B_ERR_INVALID_ARG = -1,   /* NULL pointer, token/pos out of range, bad size          */
    L2B_ERR_UNSUPPORTED = -2,   /* shape the kernels do not cover (see l2b_create)          */
    L2B_ERR_CUDA = -3,          /* a CUDA runtime call failed; see l2b_last_error()         */
    L2B_ERR_NO_DEVICE = -4,     /* no CUDA device / not compute capability 10.x             */
    L2B_ERR_OOM = -5,           /* device or pinned-host allocation failed                  */
    L2B_ERR_COMM = -6,          /* peer-memory setup failed, or a tensor-parallel peer timed out */
    L2B_ERR_STATE = -7          /* call order violated (e.g. pos beyond what was appended)  */
} l2b_status;

/* Mirrors ConfigReader (src/main.zig:17-25) after main() has normalised it (:942-946):
 * vocab_size is already abs(), shared_weights = (header vocab_size > 0).                 */
typedef struct l2b_config {
    int32_t dim;            /* transformer dimension                                       */
    int32_t hidden_dim;     /* ffn hidden dimension                                        */
    int32_t n_layers;
    int32_t n_heads;
    int32_t n_kv_heads;     /* < n_heads for multi-query / grouped-query (:291, :314-320)  */
    int32_t vocab_size;
    int32_t seq_len;
    int32_t shared_weights; /* 1: classifier == token embedding table (:112)               */
} l2b_config;

/* Tensor-parallel placement of one context (BASELINE.json config 5; SURVEY.md 8e).
 * world_size == 1 means the whole model on `device`.  For world_size in {2,4,8}
 * wq/wk/wv/w1/w3/wcls are split by output rows, wo/w2 by input columns, and the hidden
 * vector is all-reduced after wo and after w2 (inside the GEMV kernels, over NVLink peer
 * memory).  Two ways to get there:
 *   - ONE process, l2b_create(..., n_gpus): what the Zig CLI uses (`--gpus N`); nothing else
 *     changes for the caller, every l2b_* call drives all GPUs;
 *   - one process PER GPU, l2b_create_sharded with this struct: the caller moves `comm_id` (from
 *     l2b_comm_unique_id on rank 0) to every rank by its own means (bench.py uses
 *     torch.distributed) and every rank makes the same calls in the same order (lockstep: each
 *     decode step exchanges data with every other rank; a rank that stops stepping makes the
 *     others return L2B_ERR_COMM after a bounded wait, L2B_SPIN_TIMEOUT_MS, default 20 s).      */
typedef struct l2b_shard {
    int32_t rank;
    int32_t world_size;
    int32_t device;          /* CUDA device ordinal for this context                        */
    int32_t reserved;
    uint8_t comm_id[128];    /* opaque rendezvous token; ignored when world_size == 1       */
} l2b_shard;

typedef struct l2b_ctx l2b_ctx;

/* ---- lifecycle ---------------------------------------------------------------------- */

/* Replaces Weights.init (src/main.zig:73-115) + RunState.init (:137-154) on the device.
 *   host_weights : the checkpoint payload after the 28-byte header, exactly the `data`
 *                  buffer of src/main.zig:955-967, laid out as :85-112; n_floats its length.
 *   rope_cos/sin : optional (seq_len, head_size/2) tables the host computed with the
 *                  expressions of :338-342 (so RoPE is bit-identical to the host's libm);
 *                  NULL => the library computes them with the same expressions.
 *   n_gpus       : 1, 2, 4 or 8 GPUs (devices 0..n_gpus-1) driven by this one process; for
 *                  n_gpus > 1 the model is sharded as described at l2b_shard and the GPUs must
 *                  be NVLink peers.  The upload streams through pinned double buffers
 *                  (see l2b_load_stats).
 * Supported shapes: dim % 4 == 0, hidden_dim % 4 == 0, head_size = dim/n_heads a multiple of
 * 4 and <= 256, n_heads % n_kv_heads == 0; for n_gpus > 1 also n_kv_heads, hidden_dim/4 and
 * vocab_size/2 divisible by n_gpus.  Anything else => L2B_ERR_UNSUPPORTED.  Two shared-memory
 * limits are also refused here with L2B_ERR_UNSUPPORTED and a message:
 *   - a GEMV input that does not fit in shared memory: hidden_dim > 57600 on H100, or
 *     dim > 28800 where the rmsnorm gain is staged next to it;
 *   - a seq_len whose timeline split (seq_len / nsplit, at most 32 splits) no longer fits the
 *     3-pass attention kernel's 200 KB score buffer: seq_len > 1,605,632 with 8 heads or fewer.
 * DESIGN.md §4.5c tabulates which kernel runs at which limit.                              */
int32_t l2b_create(l2b_ctx **out, const l2b_config *cfg, const float *host_weights,
                   uint64_t n_floats, const float *rope_cos, const float *rope_sin,
                   int32_t n_gpus);

/* Same, for one tensor-parallel rank.  host_weights is the FULL payload; the library
 * uploads only this rank's slices.                                                         */
int32_t l2b_create_sharded(l2b_ctx **out, const l2b_config *cfg, const float *host_weights,
                           uint64_t n_floats, const float *rope_cos, const float *rope_sin,
                           const l2b_shard *shard);

/* Synthetic checkpoint of the given shape generated directly in device memory
 * (SURVEY.md 8d: stories110M / llama2-7B are not shipped; a 27 GB file is impractical).
 * The generator is a counter-based integer hash, bit-identical to
 * l2b_synth_fill_host() below, so a CPU checker can materialise the same weights.
 * shard may be NULL (single GPU, device 0).                                                */
int32_t l2b_create_synthetic(l2b_ctx **out, const l2b_config *cfg, uint64_t seed,
                             const l2b_shard *shard);
/* Same weights, one process driving n_gpus GPUs (the synthetic twin of l2b_create(.., n_gpus)). */
int32_t l2b_create_synthetic_group(l2b_ctx **out, const l2b_config *cfg, uint64_t seed,
                                   int32_t n_gpus);

/* A new decode stream on the weights of `model` (any context of it, or any session of it), with no
 * upload: its own KV cache, run state, control block, stream and graphs.  Every entry point that
 * takes a context accepts a session, and a session steps exactly as a context of the same weights
 * would.  The weights are freed when the last context or session of the model is destroyed, in
 * any order.  Single-GPU models only: a tensor-parallel model => L2B_ERR_UNSUPPORTED.
 * l2b_load_stats of a session reports 0 bytes.  A model and its sessions are not thread-safe:
 * drive them from one thread, as one context.                                              */
int32_t l2b_create_session(l2b_ctx **out, l2b_ctx *model);

void l2b_destroy(l2b_ctx *ctx);

/* Forget the KV cache (start a new generation at pos 0).  The reference runs one
 * generation per process and has no such entry point; benches need it.                     */
int32_t l2b_reset(l2b_ctx *ctx);

/* ---- the hot path ------------------------------------------------------------------- */

/* transformer(token, pos, ...) of src/main.zig:285-430.  On return host_logits[0..vocab)
 * holds what the reference leaves in state.logits (:429); the caller may then mutate it
 * exactly as :1002-1013 do.  pos must be 0 on the first call and may not skip ahead:
 * pos <= (number of positions appended so far).  Synchronous.                               */
int32_t l2b_forward(l2b_ctx *ctx, int32_t token, int32_t pos, float *host_logits);

/* Same step, but the argmax of :715-726 (first maximum wins) runs on the device in the
 * classifier epilogue and only the token id crosses PCIe.  The `-t 0` path (:1002-1003).   */
int32_t l2b_forward_argmax(l2b_ctx *ctx, int32_t token, int32_t pos, int32_t *next);

/* Zero-copy variant: runs the step and returns a pointer to the library's pinned host
 * buffer of vocab_size logits (valid until the next call on this context).                 */
int32_t l2b_forward_pinned(l2b_ctx *ctx, int32_t token, int32_t pos, const float **logits);

/* The library's pinned logits buffer (vocab_size floats, lives as long as the context).  A host
 * that uses it AS state.logits (src/main.zig:149: `state.logits = l2b_logits_buffer(ctx)[0..V]`)
 * and passes it to l2b_forward gets the logits with no second host copy: the D2H DMA of the step
 * lands directly in it.                                                                    */
float *l2b_logits_buffer(l2b_ctx *ctx);

/* transformer() + the vocab-wide part of temperature sampling (src/main.zig:1005-1012) on the
 * device: logits /= temperature (:1006), softmax (:1008), and for 0 < top_p < 1 the candidate
 * prefilter of sample_top_p (:761-768: prob >= (1-top_p)/(n-1), in index order).  The random
 * draw, the sort of the few candidates and the CDF walk stay on the host (they use the host's
 * PRNG, :730, :788).
 *   host_probs : vocab_size probabilities (what :1008 leaves in state.logits); may be NULL when
 *                only the candidates are wanted, or l2b_logits_buffer(ctx) for zero copy.
 *   cand/n_cand: for 0 < top_p < 1: *n_cand candidates (prob, index); if more than cand_cap (or
 *                8192) passed the filter, *n_cand = -(their number) and the host filters
 *                host_probs itself.  Ignored (may be NULL) for top_p == 0 or 1 (:1009).
 * vocab_size 1 => L2B_ERR_INVALID_ARG, as for l2b_op_sample_prep (the cutoff divides by n-1).  */
typedef struct l2b_prob_index { float prob; int32_t index; } l2b_prob_index;
int32_t l2b_forward_sample(l2b_ctx *ctx, int32_t token, int32_t pos, float temperature, float top_p,
                           float *host_probs, l2b_prob_index *cand, int32_t cand_cap,
                           int32_t *n_cand);

/* Whole temperature-0 generation loop of src/main.zig:995-1042 on the device: starts from
 * `token` at position `pos`, runs up to n_steps steps, feeds forced[i] (if forced != NULL
 * and forced[i] >= 0, like prompt forcing :999-1000) or the on-device argmax back in, and
 * stops after emitting BOS (token 1, :1017-1019) when stop_on_bos != 0.  out_next[i] is the
 * token chosen at step i; *n_done the number of transformer steps executed.  At most
 * seq_len - pos steps run (:992-993).  A forced entry that is read and lies outside
 * [-1, vocab_size) => L2B_ERR_INVALID_ARG before anything runs.                            */
int32_t l2b_generate_argmax(l2b_ctx *ctx, int32_t token, int32_t pos, int32_t n_steps,
                            const int32_t *forced, int32_t stop_on_bos, int32_t *out_next,
                            int32_t *n_done);

/* Prompt prefill (SURVEY.md 8f.2).  The reference feeds prompt tokens through transformer() one at
 * a time and discards their logits (src/main.zig:996-1000).  This runs positions pos0 ..
 * pos0+n_tokens-1 with tokens[i] at position pos0+i back to back on the device: no host round trip
 * per position, and the classifier is skipped for every position whose logits nobody reads.
 * host_logits == NULL: no logits at all (the KV cache is all the caller wants); otherwise the
 * logits of the LAST position are returned, exactly as l2b_forward would.  Per position the
 * arithmetic is the decode step's own, so KV cache and logits equal n_tokens calls of
 * l2b_forward bit for bit.                                                                 */
int32_t l2b_prefill(l2b_ctx *ctx, const int32_t *tokens, int32_t n_tokens, int32_t pos0,
                    float *host_logits);

/* Log-probabilities of a known sequence (teacher forcing: perplexity, reranking, comparing two
 * checkpoints).  Runs tokens[i] at position pos0+i for i = 0 .. n_tokens-2 and writes, for each i,
 *   logprob[i] = log softmax(logits at pos0+i)[tokens[i+1]]   (temperature 1, natural log)
 *   greedy[i]  = argmax of those logits, first maximum wins (:715-726)   -- greedy may be NULL
 * Afterwards the context has pos0 + n_tokens - 1 positions appended; the caller may continue with
 * l2b_forward(ctx, tokens[n_tokens-1], pos0 + n_tokens - 1, ..).  Everything is checked before
 * anything runs, so a refused call changes no KV cache: NULL ctx, tokens or logprob, n_tokens < 1,
 * a token outside [0, vocab_size), pos0 < 0 or pos0 + n_tokens - 1 > seq_len => L2B_ERR_INVALID_ARG;
 * pos0 past the positions appended => L2B_ERR_STATE; a tensor-parallel context (each rank holds only
 * a slice of the vocabulary) => L2B_ERR_UNSUPPORTED.  n_tokens == 1 runs and writes nothing.  Works on
 * any single-GPU context or session.
 * Where l2b_prefill shares weight passes, the positions run in l2b_prefill's groups of 4 (the KV rows
 * are those of l2b_prefill(tokens, n_tokens - 1, pos0) bit for bit) with the batched classifier after
 * each group; the logits are the batched prefill's, within 1e-6 (relative to the largest logit) of
 * single steps, so logprob is within 2e-6 x max|logit| + 1e-5 of the log-softmax of l2b_forward's
 * logits.  Elsewhere each position runs l2b_forward_argmax's own decode step on the device: logprob[i]
 * equals l2b_op_logprob of l2b_forward's logits bit for bit, and greedy[i] equals l2b_forward_argmax.
 * Against the exact log-softmax of the same float32 logits: within 1e-5 + 1e-6 x |logprob|.
 * Synchronous; l2b_last_timing(ctx) gives the call's device time and kernel launches.  x, xb, hb, q and
 * logits are not defined afterwards.                                                        */
int32_t l2b_score(l2b_ctx *ctx, const int32_t *tokens, int32_t n_tokens, int32_t pos0,
                  float *logprob, int32_t *greedy);

/* One transformer() step for each of n distinct sessions of one model (l2b_create_session; the
 * model's own context counts as one): sessions[i] runs tokens[i] at pos[i], under l2b_forward's rule
 * pos[i] <= (positions appended to that session).  host_logits[i] receives session i's logits.
 * On the shapes where l2b_prefill shares weight passes (bandwidth-bound, single GPU; not with
 * L2B_PREFILL_BATCH=0), up to 4 sessions share each pass over the weights, and the logits and KV
 * rows then match n l2b_forward calls to within float rounding (1e-6 relative), not bit for bit.
 * Elsewhere the sessions are stepped one after another with l2b_forward's own kernels (bit for bit).
 * Everything is checked before anything runs: n < 1, a NULL entry, the same session twice,
 * sessions of different models, a token or position out of range => L2B_ERR_INVALID_ARG; a position
 * past a session's appended count => L2B_ERR_STATE.  A refused call changes no session.  Errors
 * are reported through l2b_last_error(sessions[0]) (l2b_last_error(NULL) when there is no
 * sessions[0]), and l2b_last_timing(sessions[0]) gives the call's device time and kernel launches.
 * Afterwards l2b_read_state of each session returns its own x, key/value cache and logits, as after
 * l2b_forward; xb, hb and q are not defined after a batched step.  Synchronous.             */
int32_t l2b_forward_batch(l2b_ctx *const *sessions, int32_t n, const int32_t *tokens,
                          const int32_t *pos, float *const *host_logits);
/* Same step with the device argmax (first maximum wins, :715-726): next[i] for session i.      */
int32_t l2b_forward_argmax_batch(l2b_ctx *const *sessions, int32_t n, const int32_t *tokens,
                                 const int32_t *pos, int32_t *next);
/* Same step with l2b_forward_sample's device sampler preparation.  For each i it does what
 * l2b_forward_sample(sessions[i], tokens[i], pos[i], temperature[i], top_p[i], host_probs[i],
 * cand + i*cand_cap, cand_cap, &n_cand[i]) does: temperature and top-p are per session, cand is
 * row-major n x cand_cap, and n_cand[i] follows the single call's rule (the count, 0 when session i
 * does not filter, minus the number that passed when more than min(cand_cap, 8192) did).
 * host_probs, or any entry of it, may be NULL (those probabilities are not copied out); cand and
 * n_cand may be NULL only when no session filters (top_p 0 or 1).  Where the sessions share weight
 * passes, the sampler runs on the batched logits, so the probabilities match l2b_forward_sample to
 * float rounding; elsewhere each session runs l2b_forward_sample's own step (bit for bit).  Checked
 * before anything runs, as l2b_forward_batch, plus NULL temperature or top_p, a temperature not > 0,
 * a top_p outside [0, 1], a vocabulary of fewer than 2 entries, and a filtering session without a
 * candidate buffer or with cand_cap <= 0 => L2B_ERR_INVALID_ARG.  Afterwards l2b_read_state(..,
 * logits) of each session returns its probabilities; xb, hb and q are not defined.  Synchronous. */
int32_t l2b_forward_sample_batch(l2b_ctx *const *sessions, int32_t n, const int32_t *tokens,
                                 const int32_t *pos, const float *temperature, const float *top_p,
                                 float *const *host_probs, l2b_prob_index *cand, int32_t cand_cap,
                                 int32_t *n_cand);
/* Several positions of a session in one call: prompt chunks and decode steps of n distinct sessions
 * share weight passes.  Session i runs its n_tokens[i] >= 1 tokens at positions pos0[i] ..
 * pos0[i] + n_tokens[i] - 1; tokens holds every session's tokens back to back, in session order.
 * Each session gets one output, for its LAST position: what l2b_forward_batch, _argmax_batch or
 * _sample_batch returns for it (host_logits[i]; next[i]; probabilities, candidates and n_cand[i] under
 * the sample batch call's rules).  n_tokens[i] == 1 is a decode step, a larger count a prompt chunk or
 * a whole prompt; with every n_tokens[i] == 1 each call is its *_batch call.
 * Where l2b_prefill shares weight passes, the positions of all runs, concatenated in session order, go
 * 4 per pass (a run may straddle passes), each on its own session's cache at its own position, and
 * the classifier runs on a pass only when it holds some run's last position.  A position's arithmetic
 * does not depend on the others in its pass: a run's KV rows are those of l2b_prefill of the same
 * tokens bit for bit, its output is that of l2b_prefill of all but its last token followed by
 * l2b_forward_batch of the last one, and a prompt gives the same bits however it is cut into chunks.
 * Elsewhere each session runs l2b_prefill of all but its last token (no logits) and then its own
 * single step of the last one: bit for bit those calls.
 * Checked before anything runs, so a refused call changes no session: everything l2b_forward_batch
 * checks, plus NULL n_tokens or pos0, n_tokens[i] < 1, pos0[i] + n_tokens[i] > seq_len, a token out of
 * range anywhere in a run and a total token count past INT32_MAX => L2B_ERR_INVALID_ARG; pos0[i] past
 * the session's appended count => L2B_ERR_STATE; the sample call also makes l2b_forward_sample_batch's
 * own checks.  Errors through l2b_last_error(sessions[0]); l2b_last_timing(sessions[0]) gives the whole
 * call's device time and kernel launches.  Afterwards session i has max(its appended count, pos0[i] +
 * n_tokens[i]) positions appended, and l2b_read_state returns the x and logits (or probabilities) of its
 * last position; xb, hb and q are not defined.  Synchronous.                                   */
int32_t l2b_forward_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens,
                           const int32_t *tokens, const int32_t *pos0, float *const *host_logits);
int32_t l2b_forward_argmax_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens,
                                  const int32_t *tokens, const int32_t *pos0, int32_t *next);
int32_t l2b_forward_sample_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens,
                                  const int32_t *tokens, const int32_t *pos0,
                                  const float *temperature, const float *top_p, float *const *host_probs,
                                  l2b_prob_index *cand, int32_t cand_cap, int32_t *n_cand);
/* The greedy loop of l2b_generate_argmax on n sessions in one call, with no host round trip per
 * step.  For each i it does what l2b_generate_argmax(sessions[i], tokens[i], pos[i], n_steps,
 * forced + i*n_steps, stop_on_bos, out_next + i*n_steps, &n_done[i]) does: forced (may be NULL)
 * and out_next are row-major n x n_steps, forced[i*n_steps + s] >= 0 replaces session i's argmax at
 * step s and -1 lets it run free; session i runs at most min(n_steps, seq_len - pos[i]) steps and,
 * with stop_on_bos, stops after emitting BOS while the others go on.  Afterwards session i has
 * pos[i] + n_done[i] positions appended; its KV rows from there on are untouched.  The sessions
 * share weight passes exactly where l2b_forward_batch does, with the same kernels (up to 4 per
 * pass, all steps enqueued at once); elsewhere each session replays its own device loop on its own
 * stream, bit for bit l2b_generate_argmax.  Checked before anything runs, as l2b_forward_batch,
 * plus n_steps < 0, a NULL out_next or n_done, and a forced entry that is read and lies outside
 * [-1, vocab_size) => L2B_ERR_INVALID_ARG.  n_steps == 0 sets every n_done[i] = 0 and runs
 * nothing.  l2b_last_timing(sessions[0]) gives the whole call's device time and kernel launches.
 * x, xb, hb, q and logits of the sessions are not defined afterwards.  Synchronous.           */
int32_t l2b_generate_argmax_batch(l2b_ctx *const *sessions, int32_t n, const int32_t *tokens,
                                  const int32_t *pos, int32_t n_steps, const int32_t *forced,
                                  int32_t stop_on_bos, int32_t *out_next, int32_t *n_done);

/* ---- introspection ------------------------------------------------------------------- */

const char *l2b_last_error(const l2b_ctx *ctx);     /* never NULL                           */
const char *l2b_status_string(int32_t status);
int32_t l2b_abi_version(void);

/* Copies one RunState buffer (src/main.zig:119-135) of the last step to the host, for
 * layer-level parity tests: 0=x 1=xb 2=hb 3=q 4=key_cache 5=value_cache 6=logits.
 * Sharded contexts return this rank's slice.  n = capacity of dst in floats; *n_out the
 * floats written.                                                                          */
int32_t l2b_read_state(l2b_ctx *ctx, int32_t which, float *dst, uint64_t n, uint64_t *n_out);

/* Device time (ms, CUDA events on the context's stream) of the last l2b_generate_argmax /
 * l2b_prefill call (single steps are only timed when L2B_TIME_STEPS=1 is in the environment
 * at create time: the two event records cost the end-to-end loop of a small model ~3 %), and how
 * many kernels of this library the last call launched.                                      */
int32_t l2b_last_timing(const l2b_ctx *ctx, float *device_ms, int32_t *kernel_launches);

/* Checkpoint ingest of the last l2b_create on this context (SURVEY.md 8f.3): wall time of the
 * pinned, double-buffered upload of all weight tensors and the bytes it moved (rank 0's shard
 * for multi-GPU contexts).                                                                  */
int32_t l2b_load_stats(const l2b_ctx *ctx, double *upload_ms, uint64_t *upload_bytes);

/* Per-kernel device times of ONE step (eager launches with a CUDA event between kernels, on
 * the context's stream), for roofline accounting: `bytes` is the algorithmic traffic of that
 * launch (weight rows x columns x 4, or the K and V rows attention reads).  The step is a
 * real step (KV cache is appended, logits are produced).  out has room for cap entries;
 * *n_out receives the number of kernels in a step.                                          */
typedef struct l2b_kernel_time {
    char name[24];          /* "qkv_rope", "attention", "wo", "w13_silu", "w2", "classifier" */
    int32_t layer;          /* -1 for the classifier                                         */
    float ms;
    uint64_t bytes;
} l2b_kernel_time;
int32_t l2b_profile_step(l2b_ctx *ctx, int32_t token, int32_t pos, l2b_kernel_time *out,
                         int32_t cap, int32_t *n_out);

/* Debug: with L2B_TRACE=1 in the environment at l2b_create time, every kernel of a step stamps
 * %globaltimer at fixed points (entry, ring filled, dependency wait done, activations staged,
 * first/last stage consumed, producer done, epilogue done: slots 0..7, ns); the TMA-ring GEMV
 * also records the SM each CTA ran on (slot 8).  Copies the last step's table
 * [launch][512 CTAs][16 slots] to dst.                                                      */
int32_t l2b_debug_trace(l2b_ctx *ctx, unsigned long long *dst, uint64_t cap_words, uint64_t *n_words);

/* Algorithmic bytes one step at position pos must read (SURVEY.md 8d):
 * weight bytes (this rank's shard) and KV-cache bytes.                                     */
int32_t l2b_step_bytes(const l2b_ctx *ctx, int32_t pos, uint64_t *weight_bytes,
                       uint64_t *kv_bytes);

/* ---- multi-GPU rendezvous -------------------------------------------------------------- */
int32_t l2b_comm_unique_id(uint8_t id[128]);

/* ---- synthetic-weight generator, host mirror (for checkers) ---------------------------- */
/* dst[j] = element (first + j) of a tensor with the given seed/distribution; identical to
 * what l2b_create_synthetic puts on the device.                                            */
void l2b_synth_fill_host(float *dst, uint64_t first, uint64_t count, uint64_t tensor_seed,
                         double mean, double sigma, float lo, float hi);
/* Whole payload in checkpoint order (src/main.zig:85-112).                                 */
int32_t l2b_synth_checkpoint_host(const l2b_config *cfg, uint64_t seed, float *data,
                                  uint64_t n_floats);
uint64_t l2b_checkpoint_floats(const l2b_config *cfg);

/* ---- single ops with HOST buffers (unit-test surface) ---------------------------------- */
/* Each runs the same device code the hot path uses, on cuda:`device`, so the reference's
 * own unit tests (src/main.zig:1078-1150) can be replayed against the GPU.                 */
/* matmul (src/main.zig:485-498): xout(d) = W(d,n) . x(n)                                   */
int32_t l2b_op_matmul(int32_t device, float *xout, const float *x, const float *w, int32_t d,
                      int32_t n);
/* The fused pieces of the hot path in isolation: xout(d) = W(d,n) . rmsnorm(x, gamma) (gamma NULL
 * => W . x) through one GEMV kernel flavour (kernel: 0 = the library's own choice, 1 = latency
 * kernel, 2 = register-fed 8-row streaming kernel, 3 = TMA-ring streaming kernel).  With
 * resid_inout != NULL the result is instead accumulated into it (the residual add of :395/:422
 * in the epilogue) and xout is ignored.                                                    */
int32_t l2b_op_fused_matmul(int32_t device, float *xout, const float *x, const float *gamma,
                            const float *w, float *resid_inout, int32_t d, int32_t n,
                            int32_t kernel);
/* rmsnorm (:432-468)                                                                       */
int32_t l2b_op_rmsnorm(int32_t device, float *o, const float *x, const float *w, int32_t n);
/* softmax (:687-706), in place                                                             */
int32_t l2b_op_softmax(int32_t device, float *x, int32_t n);
/* vector_weighted_sum_rows (:657-685)                                                      */
int32_t l2b_op_weighted_sum_rows(int32_t device, float *xout, int32_t out_len, const float *rows,
                                 int32_t row_stride, const float *weights, int32_t n_weights);
/* One attention head over a KV cache slice (:361-389): q(head_size), keys/values are
 * (n_pos, kv_stride) row-major with the head's slice starting at column 0.                 */
int32_t l2b_op_attention_head(int32_t device, float *out, const float *q, const float *keys,
                              const float *values, int32_t head_size, int32_t kv_stride,
                              int32_t n_pos);

/* Sampler preparation alone (:1005-1008, :761-768) on n host logits, in place (see
 * l2b_forward_sample); *n_cand = number that passed the filter (-1 when top_p is 0 or 1).   */
int32_t l2b_op_sample_prep(int32_t device, float *logits_inout, int32_t n, float temperature,
                           float top_p, l2b_prob_index *cand, int32_t cand_cap, int32_t *n_cand);
/* log softmax(logits)[target] of n host logits (l2b_score's device code, see there).  NULL pointers,
 * n < 1 or a target outside [0, n) => L2B_ERR_INVALID_ARG.                                  */
int32_t l2b_op_logprob(int32_t device, const float *logits, int32_t n, int32_t target, float *logprob);

#ifdef __cplusplus
}
#endif
#endif /* LLAMA2_B200_H */
