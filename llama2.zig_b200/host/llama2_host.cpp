// llama2_host.cpp — see llama2_host.h.  Host-side only: no arithmetic of the hot path lives
// here; transformer() is always the l2b_* call into the CUDA library.
#include "llama2_host.h"

#include <immintrin.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <deque>
#include <string>
#include <unordered_map>
#include <vector>

// ---------------------------------------------------------------------------------------
// checkpoint (src/main.zig:936-967)
// ---------------------------------------------------------------------------------------
extern "C" int32_t l2h_load_checkpoint(const char *path, l2h_checkpoint *out) {
    if (!path || !out) return L2B_ERR_INVALID_ARG;
    memset(out, 0, sizeof *out);
    FILE *f = fopen(path, "rb");
    if (!f) return L2B_ERR_INVALID_ARG;
    int32_t h[7];
    if (fread(h, sizeof(int32_t), 7, f) != 7) { fclose(f); return L2B_ERR_INVALID_ARG; }
    l2b_config &c = out->config;
    c.dim = h[0]; c.hidden_dim = h[1]; c.n_layers = h[2]; c.n_heads = h[3]; c.n_kv_heads = h[4];
    c.shared_weights = h[5] > 0 ? 1 : 0;                 // :943
    c.vocab_size = h[5] < 0 ? -h[5] : h[5];              // :944
    c.seq_len = h[6];
    fseek(f, 0, SEEK_END);
    const long size = ftell(f);
    fseek(f, 28, SEEK_SET);
    out->n_floats = (uint64_t)(size - 28) / 4;
    out->data = (float *)malloc(out->n_floats * sizeof(float));
    if (!out->data) { fclose(f); return L2B_ERR_OOM; }
    const size_t got = fread(out->data, sizeof(float), out->n_floats, f);
    fclose(f);
    if (got != out->n_floats) { l2h_free_checkpoint(out); return L2B_ERR_INVALID_ARG; }
    return L2B_OK;
}

extern "C" void l2h_free_checkpoint(l2h_checkpoint *ck) {
    if (ck && ck->data) { free(ck->data); ck->data = nullptr; }
}

// ---------------------------------------------------------------------------------------
// tokenizer (src/main.zig:166-283)
// ---------------------------------------------------------------------------------------
struct l2h_tokenizer {
    std::vector<std::string> tokens;
    std::vector<float> scores;
    uint32_t max_token_len = 0;
    // SURVEY 8f.4: the reference's lookup is an O(vocab) scan per merge candidate (:208-215, the
    // author's TODO); same answers (FIRST id of a duplicated string) from a hash map
    std::unordered_map<std::string, int32_t> first_id;
};

extern "C" int32_t l2h_tokenizer_load(const char *path, int32_t vocab_size, l2h_tokenizer **out) {
    if (!path || !out || vocab_size <= 0) return L2B_ERR_INVALID_ARG;
    FILE *f = fopen(path, "rb");
    if (!f) return L2B_ERR_INVALID_ARG;
    l2h_tokenizer *t = new l2h_tokenizer();
    bool ok = fread(&t->max_token_len, 4, 1, f) == 1;                       // :186
    t->tokens.resize(vocab_size);
    t->scores.resize(vocab_size);
    for (int i = 0; ok && i < vocab_size; ++i) {                            // :188-193
        uint32_t len = 0;
        ok = fread(&t->scores[i], 4, 1, f) == 1 && fread(&len, 4, 1, f) == 1 && len < (1u << 20);
        if (ok) {
            t->tokens[i].resize(len);
            ok = len == 0 || fread(&t->tokens[i][0], 1, len, f) == len;
        }
    }
    fclose(f);
    if (!ok) { delete t; return L2B_ERR_INVALID_ARG; }
    t->first_id.reserve((size_t)vocab_size * 2);
    for (int i = 0; i < vocab_size; ++i) t->first_id.emplace(t->tokens[i], i);   // emplace keeps the first
    *out = t;
    return L2B_OK;
}
extern "C" void l2h_tokenizer_free(l2h_tokenizer *t) { delete t; }
extern "C" int32_t l2h_tokenizer_max_token_len(const l2h_tokenizer *t) { return t ? (int32_t)t->max_token_len : 0; }
extern "C" const char *l2h_tokenizer_token(const l2h_tokenizer *t, int32_t id, int32_t *len) {
    if (!t || id < 0 || id >= (int32_t)t->tokens.size()) return nullptr;
    if (len) *len = (int32_t)t->tokens[id].size();
    return t->tokens[id].data();
}
// first match wins (:208-215); O(1) instead of the reference's linear scan
extern "C" int32_t l2h_tokenizer_lookup(const l2h_tokenizer *t, const char *bytes, int32_t len) {
    auto it = t->first_id.find(std::string(bytes, (size_t)len));
    return it == t->first_id.end() ? -1 : it->second;
}

static int utf8_len(unsigned char c) {
    if (c < 0x80) return 1;
    if ((c & 0xE0) == 0xC0) return 2;
    if ((c & 0xF0) == 0xE0) return 3;
    if ((c & 0xF8) == 0xF0) return 4;
    return -1;
}

extern "C" int32_t l2h_tokenizer_encode(const l2h_tokenizer *t, const char *text, int32_t len, int32_t *out, int32_t cap) {
    if (!t || !text || !out) return L2B_ERR_INVALID_ARG;
    if (t->max_token_len * 2 > 128) return L2B_ERR_UNSUPPORTED;            // :222-225 TokensTooLong
    std::vector<int32_t> buf;
    for (int32_t idx = 0; idx < len;) {                                     // :236-245, one token per codepoint
        const int n = utf8_len((unsigned char)text[idx]);
        if (n < 0 || idx + n > len) return L2B_ERR_INVALID_ARG;
        const int32_t id = l2h_tokenizer_lookup(t, text + idx, n);
        if (id < 0) return L2B_ERR_INVALID_ARG;                             // TokenNotFound
        buf.push_back(id);
        idx += n;
    }
    while (buf.size() >= 2) {                                               // :247-278 greedy best-score merge
        float best_score = -1e10f;
        int32_t best_id = 0;
        int best_idx = -1;
        for (size_t i = 0; i + 1 < buf.size(); ++i) {
            std::string cat = t->tokens[buf[i]] + t->tokens[buf[i + 1]];
            const int32_t id = l2h_tokenizer_lookup(t, cat.data(), (int32_t)cat.size());
            if (id >= 0 && t->scores[id] > best_score) {
                best_score = t->scores[id];
                best_id = id;
                best_idx = (int)i;
            }
        }
        if (best_idx < 0) break;
        buf[best_idx] = best_id;
        buf.erase(buf.begin() + best_idx + 1);
    }
    if ((int32_t)buf.size() > cap) return L2B_ERR_INVALID_ARG;
    std::copy(buf.begin(), buf.end(), out);
    return (int32_t)buf.size();
}

// ---------------------------------------------------------------------------------------
// sampler (src/main.zig:715-798, :1002-1013)
// ---------------------------------------------------------------------------------------
// argmax (:715-726): strict '>' so the FIRST maximum wins.  Two passes (the maximum, then the first
// index that holds it) give the same answer as the reference's scalar scan; the first pass runs 8
// lanes wide where the host has AVX2 — the scalar scan is ~a third of the per-token host time of a
// stories15M step.  (NaNs never win in either form unless x[0] is NaN, as in the reference.)
__attribute__((target("avx2"))) static float max_avx2(const float *x, int32_t n) {
    __m256 m = _mm256_set1_ps(x[0]);
    int32_t i = 0;
    for (; i + 8 <= n; i += 8) m = _mm256_max_ps(_mm256_loadu_ps(x + i), m);
    float lanes[8];
    _mm256_storeu_ps(lanes, m);
    float max = lanes[0];
    for (int k = 1; k < 8; ++k) max = lanes[k] > max ? lanes[k] : max;
    for (; i < n; ++i) max = x[i] > max ? x[i] : max;
    return max;
}
__attribute__((target("avx2"))) static int32_t first_equal_avx2(const float *x, int32_t n, float v) {
    const __m256 vv = _mm256_set1_ps(v);
    int32_t i = 0;
    for (; i + 8 <= n; i += 8) {
        const int mask = _mm256_movemask_ps(_mm256_cmp_ps(_mm256_loadu_ps(x + i), vv, _CMP_EQ_OQ));
        if (mask) return i + __builtin_ctz(mask);
    }
    for (; i < n; ++i) if (x[i] == v) return i;
    return 0;
}
extern "C" int32_t l2h_argmax(const float *x, int32_t n) {
    if (__builtin_cpu_supports("avx2") && n >= 16) return first_equal_avx2(x, n, max_avx2(x, n));
    float max = x[0];
    for (int32_t i = 1; i < n; ++i) max = x[i] > max ? x[i] : max;
    for (int32_t i = 0; i < n; ++i)
        if (x[i] == max) return i;
    return 0;
}

extern "C" void l2h_softmax(float *x, int32_t n) {
    float max = x[0];
    for (int32_t i = 1; i < n; ++i) if (x[i] > max) max = x[i];
    float sum = 0.0f;
    for (int32_t i = 0; i < n; ++i) { x[i] = expf(x[i] - max); sum += x[i]; }
    for (int32_t i = 0; i < n; ++i) x[i] /= sum;
}

// xoshiro256++ seeded through splitmix64 (the generator family behind std.Random.DefaultPrng).
// The float mapping is a plain 24-bit one, so temperature > 0 streams are statistically, not
// bit-wise, the reference's.
static uint64_t g_s[4] = {0x9E3779B97F4A7C15ull, 0xBF58476D1CE4E5B9ull, 0x94D049BB133111EBull, 1};
static inline uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
static uint64_t next_u64() {
    const uint64_t result = rotl(g_s[0] + g_s[3], 23) + g_s[0];
    const uint64_t t = g_s[1] << 17;
    g_s[2] ^= g_s[0]; g_s[3] ^= g_s[1]; g_s[1] ^= g_s[2]; g_s[0] ^= g_s[3];
    g_s[2] ^= t;
    g_s[3] = rotl(g_s[3], 45);
    return result;
}
static float draw_f32() { return (float)(next_u64() >> 40) * (1.0f / 16777216.0f); }
// Coins drawn ahead of their turn (peek_f32) wait here and are handed out in order before any new draw, so
// peeking never changes which coin a sampled token gets.
static std::deque<float> g_queued;
static float next_f32() {
    if (g_queued.empty()) return draw_f32();
    const float r = g_queued.front();
    g_queued.pop_front();
    return r;
}
static float peek_f32(size_t ahead) {   // the coin next_f32 returns after `ahead` more calls
    while (g_queued.size() <= ahead) g_queued.push_back(draw_f32());
    return g_queued[ahead];
}
extern "C" void l2h_seed(uint64_t seed) {
    g_queued.clear();
    for (int i = 0; i < 4; ++i) {
        seed += 0x9E3779B97F4A7C15ull;
        uint64_t z = seed;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        g_s[i] = z ^ (z >> 31);
    }
}

extern "C" int32_t l2h_sample(const float *x, int32_t n) { return l2h_sample_r(x, n, next_f32()); }
extern "C" int32_t l2h_sample_r(const float *x, int32_t n, float r) {
    float cdf = 0.0f;
    for (int32_t i = 0; i < n; ++i) { cdf += x[i]; if (r < cdf) return i; }
    return n - 1;
}

struct IndexedF32 { uint32_t index; float value; };   // :743-750

extern "C" int32_t l2h_sample_top_p(const float *logits, int32_t n, float p, void *scratch) {
    const float cutoff = (1.0f - p) / ((float)n - 1.0f);                    // :761
    for (int32_t i = 0; i < n; ++i)   // a coin only when some entry passes the cutoff
        if (logits[i] >= cutoff) return l2h_sample_top_p_r(logits, n, p, scratch, next_f32());
    return l2h_argmax(logits, n);
}
extern "C" int32_t l2h_sample_top_p_r(const float *logits, int32_t n, float p, void *scratch, float coin) {
    IndexedF32 *idx = (IndexedF32 *)scratch;
    const float cutoff = (1.0f - p) / ((float)n - 1.0f);                    // :761
    int32_t m = 0;
    for (int32_t i = 0; i < n; ++i)
        if (logits[i] >= cutoff) { idx[m].value = logits[i]; idx[m].index = (uint32_t)i; ++m; }
    if (m == 0) return l2h_argmax(logits, n);
    std::sort(idx, idx + m, [](const IndexedF32 &a, const IndexedF32 &b) { return a.value > b.value; });
    float cumulative = 0.0f;
    int32_t cutoff_index = m - 1;
    for (int32_t i = 0; i < m; ++i) { cumulative += idx[i].value; if (cumulative > p) { cutoff_index = i; break; } }
    const float r = coin * cumulative;
    float cdf = 0.0f;
    for (int32_t i = 0; i <= cutoff_index; ++i) { cdf += idx[i].value; if (r < cdf) return (int32_t)idx[i].index; }
    return (int32_t)idx[cutoff_index].index;
}

extern "C" int32_t l2h_sample_top_p_candidates(l2b_prob_index *cand, int32_t m, float p) {
    return l2h_sample_top_p_candidates_r(cand, m, p, next_f32());
}
extern "C" int32_t l2h_sample_top_p_candidates_r(l2b_prob_index *cand, int32_t m, float p, float coin) {
    std::sort(cand, cand + m, [](const l2b_prob_index &a, const l2b_prob_index &b) { return a.prob > b.prob; });   // :771
    float cumulative = 0.0f;
    int32_t cutoff_index = m - 1;
    for (int32_t i = 0; i < m; ++i) { cumulative += cand[i].prob; if (cumulative > p) { cutoff_index = i; break; } }   // :774-781
    const float r = coin * cumulative;                                                                              // :785
    float cdf = 0.0f;
    for (int32_t i = 0; i <= cutoff_index; ++i) { cdf += cand[i].prob; if (r < cdf) return cand[i].index; }
    return cand[cutoff_index].index;
}

// <0xXX> raw byte tokens (:1055-1076)
static int raw_byte(const char *s, int len) {
    if (len != 6 || s[0] != '<' || s[1] != '0' || s[2] != 'x' || s[5] != '>') return -1;
    int byte = 0;
    for (int i = 3; i < 5; ++i) {
        const char c = s[i];
        byte *= 16;
        if (c >= '0' && c <= '9') byte += c - '0';
        else if (c >= 'a' && c <= 'f') byte += c - 'a' + 10;
        else if (c >= 'A' && c <= 'F') byte += c - 'A' + 10;
        else return -1;
    }
    if ((byte >= 32 && byte < 127) || byte == ' ' || (byte >= 9 && byte <= 13)) return byte;
    return -1;
}

extern "C" void l2h_print_token(const l2h_tokenizer *tk, int32_t token, int32_t next) {
    int32_t len = 0;
    const char *s = l2h_tokenizer_token(tk, next, &len);          // :1022-1034
    if (s) {
        if (token == 1 && len > 0 && s[0] == ' ') { ++s; --len; }
        const int b = raw_byte(s, len);
        if (b >= 0) fputc(b, stdout); else fwrite(s, 1, len, stdout);
    }
}

// ---------------------------------------------------------------------------------------
// generation loop (src/main.zig:995-1050)
// ---------------------------------------------------------------------------------------
extern "C" int32_t l2h_generate(l2b_ctx *ctx, const l2b_config *cfg, const l2h_gen_options *opt,
                                const int32_t *prompt, int32_t n_prompt, const l2h_tokenizer *tk,
                                int32_t *out_tokens, int32_t cap, l2h_gen_result *res) {
    if (!ctx || !cfg || !opt || !res) return L2B_ERR_INVALID_ARG;
    using clk = std::chrono::steady_clock;
    memset(res, 0, sizeof *res);
    const int V = cfg->vocab_size;
    // state.logits (:149).  The patched Zig host points state.logits at the library's pinned logits
    // buffer (INTEGRATION.md), so the D2H DMA of every step lands in it and no second copy is made.
    std::vector<float> own_logits;
    float *logits_p = l2b_logits_buffer(ctx);
    if (!logits_p) { own_logits.resize(V); logits_p = own_logits.data(); }
    struct { float *p; float *data() const { return p; } float &operator[](int i) const { return p[i]; } } logits{logits_p};
    std::vector<IndexedF32> indexed(V);                           // state.logits_indexed (:150)
    int seq_len = opt->n_steps == 0 ? cfg->seq_len : opt->n_steps;   // :992
    seq_len = std::max(1, std::min(seq_len, cfg->seq_len));          // :993
    int32_t token = 1, next = 0;                                  // :988 BOS
    bool timer_started = false;
    clk::time_point t_first;
    const clk::time_point t_begin = clk::now();
    int pos = 0;
    std::vector<l2b_prob_index> cand(8192);
    auto print_token = [&](int32_t nx) { if (tk) l2h_print_token(tk, token, nx); };
    if (opt->use_prefill && n_prompt > 0 && n_prompt < seq_len) {
        // positions 0 .. n_prompt-1 hold BOS, prompt[0 .. n_prompt-2]; their logits are never read (:999-1000)
        std::vector<int32_t> toks(n_prompt);
        toks[0] = token;
        for (int i = 1; i < n_prompt; ++i) toks[i] = prompt[i - 1];
        const int32_t rc = l2b_prefill(ctx, toks.data(), n_prompt, 0, nullptr);
        if (rc) return rc;
        res->h2d_bytes += 4ull * n_prompt;
        res->n_forward += n_prompt;
        for (; pos < n_prompt; ++pos) {
            next = prompt[pos];
            if (out_tokens && res->n_tokens < cap) out_tokens[res->n_tokens++] = next;
            print_token(next);
            token = next;
            if (!timer_started) { timer_started = true; t_first = clk::now(); }
        }
    }
    for (; pos < seq_len; ++pos) {                                // :995
        int32_t rc;
        const bool device_argmax = opt->use_device_argmax && opt->temperature == 0.0f && pos >= n_prompt;
        const bool device_sampler = opt->use_device_sampler && opt->temperature != 0.0f && pos >= n_prompt;
        if (device_sampler) {
            int32_t n_cand = 0;
            const bool filter = !(opt->top_p == 0.0f || opt->top_p == 1.0f);
            rc = l2b_forward_sample(ctx, token, pos, opt->temperature, opt->top_p, logits.data(), cand.data(),
                                    (int32_t)cand.size(), &n_cand);                        // :996 + :1005-1008 + :761-768
            if (rc) return rc;
            ++res->n_forward;
            res->h2d_bytes += 16; res->d2h_bytes += (uint64_t)V * 4 + (filter ? 8192ull * 8 + 4 : 0);
            if (!filter) next = l2h_sample(logits.data(), V);                              // :1010
            else if (n_cand > 0) next = l2h_sample_top_p_candidates(cand.data(), n_cand, opt->top_p);   // :770-797
            else next = l2h_sample_top_p(logits.data(), V, opt->top_p, indexed.data());     // too many candidates: host filters
            if (out_tokens && res->n_tokens < cap) out_tokens[res->n_tokens++] = next;
            if (opt->stop_on_bos && next == 1) break;
            print_token(next);
            token = next;
            if (!timer_started) { timer_started = true; t_first = clk::now(); }
            continue;
        }
        if (device_argmax) {
            rc = l2b_forward_argmax(ctx, token, pos, &next);      // :996 + :1003 on device
            res->h2d_bytes += 8; res->d2h_bytes += 4;
        } else {
            rc = l2b_forward(ctx, token, pos, logits.data());     // :996
            res->h2d_bytes += 8; res->d2h_bytes += (uint64_t)V * 4;
        }
        if (rc) return rc;
        ++res->n_forward;
        if (pos < n_prompt) {
            next = prompt[pos];                                   // :999-1000
        } else if (!device_argmax) {
            if (opt->temperature == 0.0f) {
                next = l2h_argmax(logits.data(), V);              // :1003
            } else {
                if (opt->temperature != 1.0f)
                    for (int i = 0; i < V; ++i) logits[i] /= opt->temperature;   // :1006
                l2h_softmax(logits.data(), V);                    // :1008
                next = (opt->top_p == 0.0f || opt->top_p == 1.0f)
                           ? l2h_sample(logits.data(), V)
                           : l2h_sample_top_p(logits.data(), V, opt->top_p, indexed.data());   // :1009-1012
            }
        }
        if (out_tokens && res->n_tokens < cap) out_tokens[res->n_tokens++] = next;
        if (opt->stop_on_bos && next == 1) break;                 // :1017-1019
        print_token(next);
        token = next;
        if (!timer_started) { timer_started = true; t_first = clk::now(); }   // :1038-1041
    }
    const clk::time_point t_end = clk::now();
    res->secs_total = std::chrono::duration<double>(t_end - t_begin).count();
    res->secs_after_first = timer_started ? std::chrono::duration<double>(t_end - t_first).count() : 0.0;
    if (tk) fflush(stdout);
    return L2B_OK;
}

// ---------------------------------------------------------------------------------------
// sampled speculative decoding: the device-sampler loop of l2h_generate, a round at a time
// ---------------------------------------------------------------------------------------
// One sampled token from the output of l2b_forward_sample (or a row of l2b_verify_sample_ragged) with the
// given coin, as the device-sampler loop picks it (:1009-1012).  *used: whether the token consumes the coin;
// it does not when top-p filtering leaves no candidate (then the argmax, as l2h_sample_top_p).
static int32_t sample_prepared(const float *probs, int32_t V, float top_p, l2b_prob_index *cand, int32_t n_cand,
                               IndexedF32 *scratch, float coin, bool *used) {
    *used = true;
    if (top_p == 0.0f || top_p == 1.0f) return l2h_sample_r(probs, V, coin);
    if (n_cand > 0) return l2h_sample_top_p_candidates_r(cand, n_cand, top_p, coin);
    *used = n_cand < 0;                 // < 0: more candidates than fit, the host filters the probabilities
    return l2h_sample_top_p_r(probs, V, top_p, scratch, coin);
}

// p: the target's next position, whose token is hist[p - pos]; dp: the stream positions the draft holds
// rows for (as in l2b_generate_speculative: after a round that accepted every draft, the draft never ran
// d_kk, so its next round first runs it at dp = p - 1).
extern "C" int32_t l2h_generate_speculative_sample(l2b_ctx *target, const l2b_config *cfg, l2b_ctx *draft,
                                                   const l2b_config *draft_cfg, int32_t token, int32_t pos,
                                                   int32_t n_steps, int32_t k, float temperature, float top_p,
                                                   int32_t stop_on_bos, int32_t *out_next, int32_t *n_done,
                                                   int32_t *n_rounds) {
    if (!target || !cfg || !draft || !draft_cfg || !out_next || !n_done || target == draft) return L2B_ERR_INVALID_ARG;
    if (k < 0 || k > L2B_SPECULATIVE_MAX_K || n_steps < 0) return L2B_ERR_INVALID_ARG;
    if (!(temperature > 0.0f) || !(top_p >= 0.0f && top_p <= 1.0f)) return L2B_ERR_INVALID_ARG;   // 0: l2b_generate_speculative
    const int V = cfg->vocab_size, S = cfg->seq_len;
    if (draft_cfg->vocab_size != V || draft_cfg->seq_len < S) return L2B_ERR_INVALID_ARG;
    if (token < 0 || token >= V || pos < 0 || pos >= S) return L2B_ERR_INVALID_ARG;
    if (n_steps > S - pos) n_steps = S - pos;                    // :992-993
    constexpr int kCap = 8192, kRun = L2B_SPECULATIVE_MAX_K + 1;
    std::vector<float> probs((size_t)kRun * V), dprobs(V);
    std::vector<l2b_prob_index> cand((size_t)kRun * kCap), dcand(kCap);
    std::vector<int32_t> n_cand(kRun), run, hist(1, token);
    std::vector<IndexedF32> scratch(V);
    int p = pos, dp = pos, done = 0, rounds = 0;
    bool stopped = false, used = false;
    int32_t rc;
    while (done < n_steps && !stopped) {
        const int kk = std::min(std::min(k, n_steps - done - 1), S - 1 - p);
        run.assign(1, hist[p - pos]);
        if (kk > 0) {
            if (dp < p && (rc = l2b_prefill(draft, hist.data() + (dp - pos), p - dp, dp, nullptr))) return rc;
            // draft token j takes the coin the stream's token at p + j + 1 would take if every draft before
            // it is accepted; the coins stay queued for the target's walk
            size_t ahead = 0;
            for (int j = 0; j < kk; ++j) {
                int32_t dn = 0;
                rc = l2b_forward_sample(draft, run.back(), p + j, temperature, top_p, dprobs.data(), dcand.data(), kCap, &dn);
                if (rc) return rc;
                run.push_back(sample_prepared(dprobs.data(), V, top_p, dcand.data(), dn, scratch.data(), peek_f32(ahead), &used));
                ahead += used;
            }
        }
        const int32_t nt = kk + 1;
        rc = l2b_verify_sample_ragged(&target, 1, &nt, run.data(), &p, &temperature, &top_p, probs.data(), cand.data(),
                                      kCap, n_cand.data());
        if (rc) return rc;
        ++rounds;
        // the plain loop's tokens: the target's own sampler and coins, in order, while it agrees with the drafts
        int emit = 0;
        for (int j = 0; j <= kk; ++j) {
            const int32_t g = sample_prepared(probs.data() + (size_t)j * V, V, top_p, cand.data() + (size_t)j * kCap,
                                              n_cand[j], scratch.data(), peek_f32(0), &used);
            if (used) next_f32();
            out_next[done + emit++] = g;
            hist.push_back(g);
            if (stop_on_bos && g == 1) { stopped = true; break; }   // :1017-1019
            if (j == kk || run[j + 1] != g) break;
        }
        if (kk > 0) dp = p + std::min(emit, kk);
        done += emit;
        p += emit;
    }
    const int end = pos + done;
    if (dp < end && (rc = l2b_prefill(draft, hist.data() + (dp - pos), end - dp, dp, nullptr))) return rc;
    *n_done = done;
    if (n_rounds) *n_rounds = rounds;
    return L2B_OK;
}
