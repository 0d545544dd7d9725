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
 *     3-pass attention kernel's 200 KB score buffer: seq_len > 1,605,632 with 8 heads or fewer;
 *     with L2B_KV_PAGED the split's page addresses follow the buffer: seq_len > 1,556,832.
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

/* Fork a shared prompt: copies rows [0, n_pos) of src's key cache and value cache, in every layer, into
 * each of the n_dst distinct sessions dst[i] of the same model (l2b_create_session; the model's own
 * context counts as one).  Afterwards each dst[i] has exactly n_pos positions appended, which may be fewer
 * than it had: a fork replaces the destination's stream.  Its rows at n_pos and beyond are not written.
 * The caller continues each destination with l2b_forward(dst[i], token, n_pos, ..) or any batch call at
 * pos n_pos (the last prompt token is re-run, as after l2b_prefill without logits).  src is not changed:
 * not its caches, its appended count, its x or its logits.  x, xb, hb, q and logits of the destinations
 * are not defined afterwards.  One pass reads each source row once and writes it to up to 8 destinations.
 * n_pos == 0 launches nothing and sets every destination's appended count to 0.
 * Everything is checked before anything launches, so a refused call changes no session: NULL src or dst,
 * n_dst < 1, a NULL entry, the same destination twice, src among the destinations, a destination of another
 * model, or n_pos < 0 => L2B_ERR_INVALID_ARG; n_pos past src's appended count => L2B_ERR_STATE; a
 * tensor-parallel src => L2B_ERR_UNSUPPORTED.  Errors are reported through l2b_last_error(src)
 * (l2b_last_error(NULL) when src is NULL); l2b_last_timing(src) gives the call's device time and kernel
 * launches.  Synchronous.                                                                    */
int32_t l2b_fork(l2b_ctx *src, int32_t n_pos, l2b_ctx *const *dst, int32_t n_dst);

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

/* ---- beam search ------------------------------------------------------------------------ */

/* Most beams one l2b_beam_search call keeps.                                                            */
#define L2B_BEAM_MAX 8

/* Beam search of B = n_beams hypotheses from `token` at position `pos` of src's prompt, on a paged model
 * (L2B_KV_PAGED).  Each hypothesis holds its KV rows in the pages of one of the B sessions `beams` (distinct
 * sessions of src's model, not src; scratch during the call), and a hypothesis that continues another one
 * takes over its parent's pages by reference instead of copying its rows.
 * The rule.  K = 2B, T = min(n_steps, seq_len - pos).  live = [the empty hypothesis, c = 0], F = [] (finished).
 * At step t = 0 .. T-1:
 *   1. each live hypothesis h, in slot order, runs its last token (at t = 0: `token`) at position pos + t;
 *   2. its candidates C_h are l2b_op_logprob_topk(logits_h, K): (lp, token) pairs, rank r_h within C_h;
 *   3. all candidates form one pool; a candidate's score is fl(c_h + lp); the pool is ordered by score (larger
 *      first, in argmax_key order), then by h, then by r_h;
 *   4. the pool is walked in order, positions counted from 0: with stop_on_bos, a BOS (token 1) candidate at a
 *      position below B goes to F, which keeps its best B, and one at position B or later is dropped; every
 *      other candidate becomes the next live slot; the walk stops at B live;
 *   5. with stop_on_bos, the search ends when |F| = B and the worst normalised score in F is >=
 *      fl(c(live[0]) / (t + 1)).
 * A hypothesis's normalised score is fl(c / len) (length penalty 1; len counts its tokens, BOS included).
 * Hypotheses are ordered by larger normalised score, then larger c, then earlier creation (step, then
 * position in that step's pool).  The results are the best B of F and live.  Without stop_on_bos, BOS is an
 * ordinary token.
 * Results, best first: result i's tokens in out_tokens[i * n_steps ..][0 .. out_len[i]) (row-major
 * n_beams x n_steps), its cumulative natural-log probability in out_logprob[i], and its KV rows in beams[i],
 * which has pos + out_len[i] positions appended and continues with l2b_forward(beams[i], last token,
 * pos + out_len[i]), as after l2b_generate_argmax.  *n_run (n_run may be NULL) is the number of steps run.
 * Contract: at every step the candidates of hypothesis [y_1 .. y_t] are l2b_op_logprob_topk of the logits
 * l2b_forward_ragged returns for the run [token, y_1 .. y_t] at pos on an l2b_fork(src, pos, ..), bit for bit:
 * where l2b_forward_ragged shares weight passes, the live hypotheses go 4 per pass through the same kernels
 * (a position's arithmetic does not depend on its pass); elsewhere each runs its own single step.  So the
 * tokens, out_len, out_logprob and the rows of beams[i] below its appended count are fixed bits, for every
 * weight and KV format.
 * Pages: every beam first releases its pages and shares src's [0, ceil(pos / P)); after each selection slot j
 * takes its parent's pages; before each step a shared page the step writes into is copied first
 * (copy-on-write, as every writing call does), so src and the siblings never change; a finished hypothesis
 * keeps its pages until the end; at the end beams[i] take the results' pages and every other reference goes
 * back to the pool.
 * Refused before anything runs or changes: NULL src, beams, out_tokens, out_len or out_logprob, n_beams
 * outside [1, L2B_BEAM_MAX] or 2 * n_beams > vocab_size, a NULL, repeated or other-model beam, src among the
 * beams, a token out of range, pos < 0 or pos >= seq_len, n_steps < 0 => L2B_ERR_INVALID_ARG; pos past src's
 * appended count => L2B_ERR_STATE; a contiguous model => L2B_ERR_UNSUPPORTED: reordering hypotheses there
 * would copy O(pos) rows per beam each step (a tensor-parallel model cannot be paged, so it is refused too).
 * n_steps == 0 runs nothing, changes nothing, and sets *n_run = 0, out_len[i] = 0 and out_logprob[i] = 0.
 * When the pool limit (l2b_kv_pool_limit) or the device memory runs out at any step the call returns
 * L2B_ERR_OOM: src is unchanged, every beam has 0 positions appended and no page is lost.  This is weaker
 * than "changes no session": the beams are destinations whose streams the call replaces, as in l2b_fork.
 * src is never changed: not its caches, its appended count or its logits.  x, xb, hb, q and logits of the
 * beams are not defined afterwards.  Errors through l2b_last_error(src); l2b_last_timing(src) covers the
 * whole call, host work between the steps included.  Synchronous.                                         */
int32_t l2b_beam_search(l2b_ctx *src, int32_t token, int32_t pos, l2b_ctx *const *beams, int32_t n_beams,
                        int32_t n_steps, int32_t stop_on_bos, int32_t *out_tokens, int32_t *out_len,
                        float *out_logprob, int32_t *n_run);

/* ---- greedy speculative decoding ------------------------------------------------------ */

/* Verifies guessed ("draft") tokens of n distinct sessions in shared weight passes.  The runs are laid out
 * as in l2b_forward_argmax_ragged: run i is [t, d_1 .. d_m] at positions pos0[i] .., m = n_tokens[i] - 1,
 * where t is the session's last emitted token and d_j are drafts; off_i is the run's first entry in tokens.
 *   greedy   : the layout of tokens; greedy[off_i + j] is the argmax (first maximum wins, :715-726) at
 *              position pos0[i] + j, for j <= n_accept[i].  Entries past that are not written.
 *   n_accept : n_accept[i] is the largest a <= m such that for every j < a, d_{j+1} == greedy[off_i + j]
 *              and, with stop_on_bos, greedy[off_i + j] != 1.  The session emits greedy[off_i .. off_i + a]:
 *              a + 1 tokens, exactly those of l2b_generate_argmax_batch from (t, pos0[i]), whatever the drafts.
 * Afterwards session i has exactly pos0[i] + n_accept[i] + 1 positions appended (which may be fewer than it
 * had, as after l2b_fork); its KV rows below that equal the greedy loop's bit for bit, its rows past it are
 * not defined, nor are x, xb, hb, q and logits.  Where l2b_forward_ragged shares weight passes the vectors go
 * 4 per pass with the same kernels, and after each pass's classifier verify_accept_kernel decides the runs it
 * holds; once every run is decided the passes still queued return at once.  Elsewhere each run is a device
 * loop of single decode steps (every position runs).  With every n_tokens[i] == 1, greedy equals
 * l2b_forward_argmax_batch's next bit for bit.  Checked before anything runs, so a refused call changes no
 * session: everything l2b_forward_argmax_ragged checks, plus NULL greedy or n_accept => L2B_ERR_INVALID_ARG;
 * a tensor-parallel model => L2B_ERR_UNSUPPORTED.  Errors through l2b_last_error(sessions[0]);
 * l2b_last_timing(sessions[0]) gives the call's device time and kernel launches.  Synchronous.         */
int32_t l2b_verify_argmax_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens,
                                 const int32_t *tokens, const int32_t *pos0, int32_t stop_on_bos,
                                 int32_t *greedy, int32_t *n_accept);

/* Most drafts one round of l2b_generate_speculative proposes.                                        */
#define L2B_SPECULATIVE_MAX_K 32

/* ---- sampled speculative decoding ------------------------------------------------------ */

/* The positions one l2b_verify_sample_ragged call may run.  Every position's output crosses to the host
 * through one pinned staging area of the call: vocab_size probabilities and 8192 candidates, 4 * vocab_size
 * + 65536 bytes a position (193,536 at vocab_size 32000).  The staging may hold L2B_VERIFY_SAMPLE_STAGE_BYTES,
 * so the cap on sum(n_tokens) is
 *     max(n * (L2B_SPECULATIVE_MAX_K + 1), L2B_VERIFY_SAMPLE_STAGE_BYTES / (4 * vocab_size + 65536))
 * which is 346 positions at vocab_size 32000, and never less than a full round for every session.         */
#define L2B_VERIFY_SAMPLE_STAGE_BYTES (64 << 20)

/* The sampler preparation of l2b_forward_sample_ragged at EVERY position of the runs, for sampled speculative
 * decoding: the host walks the positions with its own sampler and coins (PRNG draws) and accepts drafts while
 * the sampled token equals the next draft.  The runs are laid out as in l2b_forward_sample_ragged (run i is
 * n_tokens[i] tokens at positions pos0[i] ..; total = sum(n_tokens)), and position v of that layout gets
 *   host_probs + v * vocab_size : its probabilities (host_probs may be NULL: none are copied),
 *   cand + v * cand_cap, n_cand[v] : its candidates and their count under l2b_forward_sample's rules (the
 *                  count; minus the number that passed when more than min(cand_cap, 8192) did; 0 when the
 *                  session does not filter).  cand and n_cand may be NULL when no session filters,
 * exactly what l2b_forward_sample_ragged returns for a run ending at that position.  Where l2b_forward_ragged
 * shares weight passes, every pass runs the classifier and sample_prep_batch_kernel over all its rows: a
 * position's arithmetic does not depend on its pass, so its outputs equal l2b_forward_sample_ragged's bit for
 * bit.  Elsewhere each position runs l2b_forward_sample's own step: bit for bit that call.
 * Afterwards session i has max(its appended count, pos0[i] + n_tokens[i]) positions appended, as after the
 * ragged call.  A host that accepts fewer positions continues at its accepted position (pos <= appended allows
 * it); the rows past that position are stale until they are overwritten.  x, xb, hb, q and logits are not
 * defined afterwards.  Checked before anything runs, so a refused call changes no session: everything
 * l2b_forward_sample_ragged checks, and a total above the cap of L2B_VERIFY_SAMPLE_STAGE_BYTES =>
 * L2B_ERR_INVALID_ARG; a tensor-parallel model => L2B_ERR_UNSUPPORTED.  Errors through
 * l2b_last_error(sessions[0]); l2b_last_timing(sessions[0]) gives the call's device time and kernel
 * launches.  Synchronous.                                                                               */
int32_t l2b_verify_sample_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens,
                                 const int32_t *tokens, const int32_t *pos0,
                                 const float *temperature, const float *top_p, float *host_probs,
                                 l2b_prob_index *cand, int32_t cand_cap, int32_t *n_cand);

/* The greedy loop of l2b_generate_argmax on `target`, a round at a time: `draft` (another context or session
 * with the same vocabulary, of any model) proposes kk = min(k, tokens still wanted - 1, seq_len - 1 - p)
 * tokens with its own device loop, and one l2b_verify_argmax_ragged of one run checks them on the target,
 * which emits the accepted ones and its own next token.  The tokens (out_next[0 .. *n_done)), *n_done and the
 * target's KV rows [0, pos + *n_done) equal those of l2b_generate_argmax_batch(&target, 1, &token, &pos,
 * n_steps, NULL, stop_on_bos, ..) bit for bit, for any draft; a BOS stop and the seq_len limit behave as
 * there.  The draft is kept in step: after a round that rejected a draft its rows already hold the accepted
 * tokens; after one that accepted all, its next loop starts one position earlier, forced through the
 * stream.  Afterwards target and draft each have exactly pos + *n_done positions appended, holding the same
 * tokens (one l2b_prefill of the draft when the last round accepted everything), so a second call from
 * (out_next[*n_done - 1], pos + *n_done) continues the stream.  k == 0 verifies one position per round.
 * *n_rounds (n_rounds may be NULL) is the number of rounds.  Checked before anything runs: NULL target,
 * draft, out_next or n_done, target == draft, k outside [0, L2B_SPECULATIVE_MAX_K], n_steps < 0, a token or
 * pos out of range, a different vocab_size or a draft seq_len below the target's => L2B_ERR_INVALID_ARG;
 * pos past either context's appended count => L2B_ERR_STATE; a tensor-parallel target or draft =>
 * L2B_ERR_UNSUPPORTED.  Errors through l2b_last_error(target); l2b_last_timing(target) covers the whole
 * call, draft included.  x, xb, hb, q and logits of both are not defined afterwards.  Synchronous.     */
int32_t l2b_generate_speculative(l2b_ctx *target, l2b_ctx *draft, int32_t token, int32_t pos,
                                 int32_t n_steps, int32_t k, int32_t stop_on_bos, int32_t *out_next,
                                 int32_t *n_done, int32_t *n_rounds);

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
/* The k best log softmax(logits)[i] of n host logits, best first: out[j] = (log-probability, index), ordered
 * by larger log-probability, then smaller index.  Each out[j].prob equals l2b_op_logprob(.., out[j].index)
 * bit for bit.  NULL pointers, n < 1, k < 1, k > n or k > 2 * L2B_BEAM_MAX => L2B_ERR_INVALID_ARG.
 * Here l2b_prob_index.prob holds a log-probability, not a probability.  The selection is on the
 * log-probabilities themselves: two logits that round to one log-probability tie, and the smaller index
 * comes first.  l2b_beam_search's candidates are this kernel's output.                                  */
int32_t l2b_op_logprob_topk(int32_t device, const float *logits, int32_t n, int32_t k, l2b_prob_index *out);

/* ---- device weight format ------------------------------------------------------------------
 * Which tensors: the token embedding, wq wk wv wo w1 w2 w3 and an unshared wcls are stored in the
 * format; the RMSNorm gains, RoPE tables, KV cache and all run state stay fp32.
 * Rounding (L2B_WEIGHTS_BF16): each fp32 weight becomes the nearest bf16, ties to even.  +-inf stays
 * +-inf, finite values above the bf16 maximum become +-inf, subnormals are rounded (not flushed), NaN
 * stays NaN.  For every non-NaN value this is bitwise torch's float32 -> bfloat16 -> float32 round
 * trip.  The host upload, l2b_round_bf16_host and the synthetic generator share this one rounding.
 * Contract: for every payload P and every entry point, a bf16 context of P (and its sessions) returns
 * exactly what an fp32 context of round_bf16(P) (P with those tensors rounded) returns: logits, probabilities, candidates,
 * log-probabilities, tokens, n_accept, n_done, and l2b_read_state of x, the KV cache and the logits.
 * Each bf16 kernel is the fp32 kernel the same shape selects, reading bf16 and widening it exactly.
 * Device rows of a bf16 matrix are padded to a multiple of 8 elements (16 bytes) with zeros.
 * l2b_load_stats, l2b_step_bytes and the bytes of l2b_profile_step count 2 bytes per bf16 element
 * stored, padding included.
 * Quantization (L2B_WEIGHTS_Q8): row r of a matrix of n columns is cut into groups of L2B_Q8_GROUP
 * weights, [64g, min(n, 64g + 64)) (the last group of a row may be short; no group spans two rows).
 * In fp32, with IEEE division and no contraction: a = max |w| over the group, s = a / 127.0f; a == 0
 * gives s = 0 and every q = 0, otherwise q = clamp(rint(w / s), -127, 127) with rint to nearest even
 * (0 / 0, when s underflows to 0, gives q = 0).  The dequantized weight is w' = fl((float)q * s), the
 * only value any kernel multiplies.  A non-finite matrix weight has no group scale and is refused with
 * L2B_ERR_INVALID_ARG (by an upload as it quantizes: the context is freed and *out stays NULL).  The
 * host upload, l2b_round_q8_host and the synthetic generator share this one quantizer.
 * Contract, as for bf16: a q8 context of P returns exactly what an fp32 context of dq(P) (P with
 * every matrix weight replaced by w') returns, for every entry point.  Each q8 kernel is the fp32
 * kernel the same shape selects; every thread rebuilds the weights of its fp32 columns as w' and adds
 * in the fp32 order.  A q8 row is stored as its n int8 codes zero-padded to 16 bytes, followed by its
 * ceil(n / 64) fp32 scales zero-padded to 16 bytes; l2b_load_stats, l2b_step_bytes and the bytes of
 * l2b_profile_step count 1 byte per stored code and 4 per stored scale, padding included.
 * Sessions (l2b_create_session) of a bf16 or q8 model share its format; l2b_create_sharded stays fp32. */
/* 2 is not a format: it stays an unknown format (L2B_ERR_INVALID_ARG), as it was before q8 existed.   */
typedef enum l2b_weight_format { L2B_WEIGHTS_F32 = 0, L2B_WEIGHTS_BF16 = 1, L2B_WEIGHTS_Q8 = 3 } l2b_weight_format;
#define L2B_Q8_GROUP 64

/* l2b_create with a device weight format (and optionally L2B_KV_BF16, see below).  L2B_WEIGHTS_F32 is
 * exactly l2b_create.  Checked before
 * any device is touched: an unknown format => L2B_ERR_INVALID_ARG; L2B_WEIGHTS_BF16 or L2B_WEIGHTS_Q8
 * with n_gpus > 1 => L2B_ERR_UNSUPPORTED (tensor parallel is fp32 only); every other check is
 * l2b_create's, plus (q8) a non-finite matrix weight => L2B_ERR_INVALID_ARG.                        */
int32_t l2b_create_format(l2b_ctx **out, const l2b_config *cfg, const float *host_weights, uint64_t n_floats,
                          const float *rope_cos, const float *rope_sin, int32_t n_gpus, int32_t weight_format);
/* l2b_create_synthetic (single GPU, device 0) with a device weight format.  The bf16 matrices are
 * exactly those of l2b_synth_checkpoint_host's payload passed through l2b_round_bf16_host, the q8
 * ones exactly a q8 upload of that payload.                                                         */
int32_t l2b_create_synthetic_format(l2b_ctx **out, const l2b_config *cfg, uint64_t seed, int32_t weight_format);
/* Format of ctx's model, and how many matrix weights rounding (bf16) or quantization (q8) changed
 * (their bit pattern differs from the fp32 value; 0: every output equals that of an fp32 context of
 * the same payload).  Counted during the upload, or on the device for synthetic weights.           */
int32_t l2b_weight_info(const l2b_ctx *ctx, int32_t *weight_format, uint64_t *n_rounded);
/* In place: each value -> the nearest bf16 (ties to even), widened back to fp32.  The library's own
 * rounding (see above).                                                                            */
void l2b_round_bf16_host(float *data, uint64_t n);
/* In place on a rows x cols row-major matrix: each weight -> its q8 dequantized value w' (see above);
 * *n_changed (if not NULL) = how many weights changed bitwise.  A stacked [L][rows][cols] tensor is
 * L * rows rows.  NULL data, cols == 0, cols > 2^30 or a non-finite value => L2B_ERR_INVALID_ARG with
 * data untouched (every value is checked before any is written).                                   */
int32_t l2b_round_q8_host(float *data, uint64_t rows, uint64_t cols, uint64_t *n_changed);

/* ---- KV-cache format ------------------------------------------------------------------------
 * L2B_KV_BF16, or'd into the weight_format of l2b_create_format / l2b_create_synthetic_format (with any
 * weight format, e.g. L2B_WEIGHTS_Q8 | L2B_KV_BF16), keeps the context's key and value caches in bf16:
 * half the cache memory and half the cache bytes attention reads per step.  Any other bit outside the
 * weight formats => L2B_ERR_INVALID_ARG; L2B_KV_BF16 with n_gpus > 1 => L2B_ERR_UNSUPPORTED (tensor
 * parallel is fp32 only), both checked before any device is touched.  Sessions (l2b_create_session)
 * take their model's KV format, so every batched call and every l2b_fork is of one format.
 * Rounding: every K value (after RoPE) and every V value is rounded to the nearest bf16, ties to even,
 * as it is appended (the weights' rounding above: NaN stays NaN, overflow goes to +-inf, subnormals are
 * rounded).  Attention widens each stored value exactly; q, scores, softmax, partials and all run state
 * stay fp32.
 * Contract: a bf16-KV context returns, on every entry point, exactly what an fp32-KV context of the same
 * payload and weight format returns when it rounds every appended K/V value to bf16 before storing it
 * (an L2B_KV_ROUND_BF16 context, below): logits,
 * probabilities, candidates, log-probabilities, tokens, n_accept, n_done, and l2b_read_state of x, the
 * KV cache and the logits.  Each bf16-KV kernel is the fp32 kernel the same shape selects.
 * l2b_read_state(4 / 5) returns the caches widened to fp32 (the same count of floats); l2b_step_bytes'
 * kv_bytes and the attention / attn_wo bytes of l2b_profile_step count 2 bytes per stored element.     */
#define L2B_KV_BF16 0x100
/* The reference of that contract, for tests: an fp32 cache that rounds every appended K/V value to bf16
 * and stores it widened; attention runs the fp32 kernels.  It is not a format to serve with: it costs the
 * fp32 cache's memory and bytes and the bf16 cache's accuracy.  Or'd in like L2B_KV_BF16, with the same
 * checks; both flags together => L2B_ERR_INVALID_ARG.                                                  */
#define L2B_KV_ROUND_BF16 0x200
/* The KV format of ctx (0: fp32, L2B_KV_BF16, L2B_KV_ROUND_BF16, L2B_KV_E4M3, L2B_KV_ROUND_E4M3) and the
 * bytes of its key and value caches together: 2 * n_layers * seq_len * kv_dim * (2 for L2B_KV_BF16, 1 for
 * L2B_KV_E4M3, else 4).  l2b_weight_info reports the
 * weight format alone.  A paged context (below) reports the element format alone, and as cache bytes the
 * pages it references times page_bytes: a page shared by several sessions counts in each of them
 * (l2b_kv_pool_info gives the true total).                                                             */
int32_t l2b_kv_info(const l2b_ctx *ctx, int32_t *kv_format, uint64_t *cache_bytes);

/* ---- Paged KV layout ------------------------------------------------------------------------
 * L2B_KV_PAGED, or'd into the weight_format of l2b_create_format / l2b_create_synthetic_format (with any
 * weight format, and with or without L2B_KV_BF16 or L2B_KV_ROUND_BF16), keeps the caches of the model's
 * contexts and sessions in pages of L2B_KV_PAGE_ROWS positions drawn from one pool per model.  A page
 * holds those positions of every layer, K and V.  A session holds only the pages of the positions it has
 * appended, and l2b_fork shares the source's full pages with its destinations instead of copying them: a
 * destination that writes into a shared page first gets a private copy (copy-on-write).  n_gpus > 1 =>
 * L2B_ERR_UNSUPPORTED, checked before any device is touched.  Sessions take their model's layout.
 * Contract: a paged context returns, on every entry point, exactly what a contiguous context of the same
 * payload, weight format and KV format returns (the outputs listed under the KV format above, and
 * l2b_read_state of the cache rows below the appended count), after any sequence of forks, rewinds,
 * resets and copies-on-write.  Its kernels are the contiguous kernels the same shape selects; only the
 * row addresses differ.
 * Changed promises of a paged context:
 *  - Every call that appends rows first reserves the pages of every row it may write.  When the pool
 *    limit (l2b_kv_pool_limit) or the device memory runs out, the call returns L2B_ERR_OOM and changes no
 *    session.  After the call, every page that lies wholly at or past a session's appended count is
 *    released, as l2b_reset releases all of them and l2b_destroy a session's.
 *  - Rows at and past the appended count are not defined, also where a contiguous context leaves them
 *    "untouched" or "not written": they may lie in a released page.
 *  - l2b_read_state(4 / 5) gathers the rows into the contiguous (L, seq_len, kv_dim) fp32 layout; rows in
 *    no page the context holds read as 0.
 *  - l2b_fork releases each destination's pages, then shares src's full pages and copies the rows of its
 *    last partial page (at most L2B_KV_PAGE_ROWS - 1 rows) into a fresh page per destination; when n_pos
 *    is a multiple of L2B_KV_PAGE_ROWS nothing is copied.                                              */
#define L2B_KV_PAGED 0x800
#define L2B_KV_PAGE_ROWS 64
/* The pool of ctx's model: rows per page, bytes per page (2 * n_layers * L2B_KV_PAGE_ROWS * kv_dim * the
 * element size), pages held by some context or session, and pages allocated on the device (in use or
 * free; free pages are kept until the model is destroyed).  Any context or session of the model; a
 * contiguous model reports zeros.  NULL ctx or any NULL output => L2B_ERR_INVALID_ARG.                */
int32_t l2b_kv_pool_info(const l2b_ctx *ctx, int32_t *page_rows, uint64_t *page_bytes, uint64_t *pages_in_use,
                         uint64_t *pages_allocated);
/* Caps the pages ctx's model may have in use (0: no cap, the default); a call that would need more returns
 * L2B_ERR_OOM and changes no session.  A cap below the pages in use => L2B_ERR_INVALID_ARG; a contiguous
 * model => L2B_ERR_UNSUPPORTED; NULL ctx => L2B_ERR_INVALID_ARG.                                       */
int32_t l2b_kv_pool_limit(l2b_ctx *ctx, uint64_t max_pages);

/* ---- fp8 (e4m3) KV cache ----------------------------------------------------------------------
 * L2B_KV_E4M3, or'd into the weight_format of l2b_create_format / l2b_create_synthetic_format (with any
 * weight format, with or without L2B_KV_PAGED), keeps the caches in OCP FP8 E4M3 ("e4m3fn": bias 7, no
 * infinities, largest finite +-448, NaN S.1111.111): a quarter of the fp32 cache's memory and bytes, half
 * the bf16 cache's.  Any two of L2B_KV_BF16, L2B_KV_ROUND_BF16, L2B_KV_E4M3 and L2B_KV_ROUND_E4M3 together
 * => L2B_ERR_INVALID_ARG; n_gpus > 1 => L2B_ERR_UNSUPPORTED; both checked before any device is touched.
 * Scales: each layer l has one fp32 scale for K, s_k[l], and one for V, s_v[l] (l2b_kv_scales; 1 by
 * default).  An appended value v (K after RoPE, or V) with its layer's scale s is stored as the code
 * c = e4m3(fl(v / s)): IEEE division, then the nearest e4m3 value, ties to even, subnormals rounded, the
 * sign of zero kept, finite values past 448 and +-inf to +-448 (saturating), NaN to NaN.  Attention reads
 * fl((float)c * s) for each element; q, scores, softmax, partials and all run state stay fp32.
 * Contract: an e4m3-KV context returns, on every entry point, exactly what an L2B_KV_ROUND_E4M3 context of
 * the same payload, weight format, layout and scales returns (the outputs listed under L2B_KV_BF16, and
 * l2b_beam_search's).  Each e4m3 kernel is the fp32 kernel the same shape selects.  l2b_read_state(4 / 5)
 * returns the caches widened with the scales (fl((float)c * s)); l2b_kv_info's cache bytes,
 * l2b_step_bytes' kv_bytes, the attention / attn_wo bytes of l2b_profile_step and l2b_kv_pool_info's
 * page_bytes count 1 byte per stored element.                                                         */
#define L2B_KV_E4M3 0x1000
/* The reference of that contract, for tests: an fp32 cache that stores fl((float)e4m3(fl(v / s)) * s) for
 * every appended value and is read by the fp32 kernels.  Not a format to serve with.                   */
#define L2B_KV_ROUND_E4M3 0x2000
/* Sets the KV scales of ctx's model: scales[2l] = s_k[l], scales[2l + 1] = s_v[l], n == 2 * n_layers.  They
 * live in the model's device memory; sessions created afterwards use them too.  Every refusal leaves the
 * scales unchanged: NULL ctx or scales, a wrong n, or a scale that is not a finite positive normal float
 * => L2B_ERR_INVALID_ARG; a model whose KV format is neither e4m3 flag => L2B_ERR_UNSUPPORTED; a model
 * with a live session, or with positions appended (rows stored under the old scales would be misread),
 * => L2B_ERR_STATE.                                                                                   */
int32_t l2b_kv_scales(l2b_ctx *ctx, const float *scales, int32_t n);
/* In place, the value an e4m3 cache element stands for: v -> fl((float)e4m3(fl(v / scale)) * scale), the
 * rounding above.  NULL data does nothing.                                                             */
void l2b_round_e4m3_host(float *data, uint64_t n, float scale);

#ifdef __cplusplus
}
#endif
#endif /* LLAMA2_B200_H */
