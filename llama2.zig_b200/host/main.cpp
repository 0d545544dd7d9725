// llama2_b200 — command-line twin of the reference's `llama2` binary (src/main.zig:823-1051)
// with transformer() served by the H100 library.  Same flags and usage text (:800-813).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <chrono>
#include <string>
#include <vector>

#include "llama2_host.h"

static const char *usage_text =
    "Usage:   llama2_b200 <checkpoint> [options]\n"
    "Example: llama2_b200 checkpoint.bin -n 256 -i \"Once upon a time\"\n"
    "Options:\n"
    " -h, --help                print this help message\n"
    " -t, --temperature <float> temperature, default 1.0 (0.0, 1]\n"
    " -p, --top-p <float>       p value in top-p (nucleus) sampling. default 0.9, 0 || 1 = off\n"
    " -n, --seq-len <int>       number of steps to run for, default 256. 0 = max_seq_len\n"
    " -i, --input <string>      input text for the prompt, default \"\"\n"
    " -s, --seed <int>          random seed, default to time\n"
    " -v, --verbose             print model info and tokens/s\n"
    " -z, --tokenizer <path>    path to the tokenizer to use, default to \"tokenizer.bin\"\n"
    "     --device-argmax       with -t 0: argmax on the GPU, only the token id crosses PCIe\n"
    "     --device-sampler      with -t > 0: logits/T, softmax and the top-p prefilter on the GPU\n"
    "     --prefill             prompt positions run on the GPU back to back (no logits, no host round trip)\n"
    "     --gpus <1|2|4|8>      tensor-parallel over that many GPUs (llama2-7B class models)\n"
    "     --draft <checkpoint>  speculative decoding with this draft model (same vocabulary); same tokens\n"
    "     --draft-k <int>       tokens the draft proposes per round, default 3, at most 32\n"
    "     --bf16                keep the matrix weights (and the draft's) in bf16 on the GPU: half the memory and\n"
    "                           bytes per step; outputs equal an fp32 run of the bf16-rounded checkpoint (1 GPU)\n"
    "     --q8                  keep the matrix weights (and the draft's) as int8 with one scale per 64 weights: 0.53x\n"
    "                           the bf16 bytes per step; outputs equal an fp32 run of the dequantized checkpoint (1 GPU)\n"
    "     --kv-bf16             keep the KV cache (and the draft's) in bf16 on the GPU: half the cache memory and\n"
    "                           attention bytes; outputs equal an fp32-cache run that rounds each K/V value (1 GPU)\n"
    "     --kv-e4m3             keep the KV cache (and the draft's) in fp8 e4m3 with unit scales: half the bf16 cache's\n"
    "                           memory; outputs equal an fp32-cache run that rounds each K/V value to e4m3 (1 GPU)\n"
    "     --beam <int>          beam search with that many hypotheses (at most 8) on a paged KV cache; prints the\n"
    "                           best one; -t and -p are ignored, -v prints every result's normalised score (1 GPU)\n";

// -v: the KV-cache format and bytes of a context (l2b_kv_info)
static void print_kv_info(const char *what, const l2b_ctx *ctx) {
    int32_t fmt = 0;
    uint64_t bytes = 0;
    l2b_kv_info(ctx, &fmt, &bytes);
    fprintf(stderr, "%s: %s, %llu bytes\n", what, fmt == L2B_KV_BF16 ? "bf16" : fmt == L2B_KV_ROUND_BF16 ? "fp32 (bf16-rounded)"
                                    : fmt == L2B_KV_E4M3 ? "e4m3" : fmt == L2B_KV_ROUND_E4M3 ? "fp32 (e4m3-rounded)" : "fp32",
            (unsigned long long)bytes);
}

// Generation with a draft model: the prompt positions are prefilled on target and draft, then
// l2b_generate_speculative (-t 0) or l2h_generate_speculative_sample (-t > 0) runs the rest.  The tokens
// are those of the --device-argmax / --device-sampler loops with the same seed, whatever the draft.
static int generate_with_draft(l2b_ctx *ctx, const l2b_config &c, l2b_ctx *draft, const l2b_config &dc, int k,
                               const l2h_gen_options &opt, const std::vector<int32_t> &prompt, const l2h_tokenizer *tk,
                               bool verbose) {
    int seq_len = opt.n_steps == 0 ? c.seq_len : opt.n_steps;   // :992-993
    seq_len = seq_len < 1 ? 1 : seq_len > c.seq_len ? c.seq_len : seq_len;
    const int n_prompt = (int)prompt.size() < seq_len ? (int)prompt.size() : seq_len;
    int32_t token = 1, rc;                                      // :988 BOS
    if (n_prompt > 0 && n_prompt < seq_len) {   // positions 0 .. n_prompt-1 hold BOS, prompt[0 .. n_prompt-2] (:999-1000)
        std::vector<int32_t> toks(1, token);
        toks.insert(toks.end(), prompt.begin(), prompt.begin() + n_prompt - 1);
        for (l2b_ctx *t : {ctx, draft})
            if ((rc = l2b_prefill(t, toks.data(), n_prompt, 0, nullptr))) return rc;
    }
    for (int i = 0; i < n_prompt; ++i) { l2h_print_token(tk, token, prompt[i]); token = prompt[i]; }
    if (n_prompt == seq_len) return L2B_OK;
    std::vector<int32_t> out(seq_len);
    int32_t done = 0, rounds = 0;
    const auto t0 = std::chrono::steady_clock::now();
    rc = opt.temperature == 0.0f
             ? l2b_generate_speculative(ctx, draft, token, n_prompt, seq_len - n_prompt, k, opt.stop_on_bos,
                                        out.data(), &done, &rounds)
             : l2h_generate_speculative_sample(ctx, &c, draft, &dc, token, n_prompt, seq_len - n_prompt, k,
                                               opt.temperature, opt.top_p, opt.stop_on_bos, out.data(), &done, &rounds);
    if (rc) return rc;
    const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    for (int i = 0; i < done; ++i) {
        if (opt.stop_on_bos && out[i] == 1) break;              // :1017-1019
        l2h_print_token(tk, token, out[i]);
        token = out[i];
    }
    fflush(stdout);
    if (verbose && secs > 0)
        fprintf(stderr, "\n\n%d tokens in %d rounds, %d tokens per second\n", done, rounds, (int)(done / secs));
    return L2B_OK;
}

// Beam search (--beam N): the prompt is prefilled as above, then l2b_beam_search runs N hypotheses on N
// sessions of the paged model to the step limit, and the best one is printed.  -t and -p play no part.
static int generate_beam(l2b_ctx *ctx, const l2b_config &c, int n_beams, const l2h_gen_options &opt,
                         const std::vector<int32_t> &prompt, const l2h_tokenizer *tk, bool verbose) {
    int seq_len = opt.n_steps == 0 ? c.seq_len : opt.n_steps;   // :992-993
    seq_len = seq_len < 1 ? 1 : seq_len > c.seq_len ? c.seq_len : seq_len;
    const int n_prompt = (int)prompt.size() < seq_len ? (int)prompt.size() : seq_len;
    int32_t token = 1, rc = L2B_OK;                             // :988 BOS
    if (n_prompt > 0 && n_prompt < seq_len) {
        std::vector<int32_t> toks(1, token);
        toks.insert(toks.end(), prompt.begin(), prompt.begin() + n_prompt - 1);
        if ((rc = l2b_prefill(ctx, toks.data(), n_prompt, 0, nullptr))) return rc;
    }
    for (int i = 0; i < n_prompt; ++i) { l2h_print_token(tk, token, prompt[i]); token = prompt[i]; }
    if (n_prompt == seq_len) return L2B_OK;
    const int n_steps = seq_len - n_prompt;
    std::vector<l2b_ctx *> beams;
    for (int i = 0; i < n_beams && rc == L2B_OK; ++i) {
        l2b_ctx *s = nullptr;
        rc = l2b_create_session(&s, ctx);
        if (s) beams.push_back(s);
    }
    std::vector<int32_t> out((size_t)n_beams * n_steps), len(n_beams);
    std::vector<float> lp(n_beams);
    int32_t ran = 0;
    const auto t0 = std::chrono::steady_clock::now();
    if (rc == L2B_OK)
        rc = l2b_beam_search(ctx, token, n_prompt, beams.data(), n_beams, n_steps, opt.stop_on_bos, out.data(),
                             len.data(), lp.data(), &ran);
    const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    for (l2b_ctx *s : beams) l2b_destroy(s);
    if (rc) return rc;
    for (int i = 0; i < len[0]; ++i) {
        if (opt.stop_on_bos && out[i] == 1) break;              // :1017-1019
        l2h_print_token(tk, token, out[i]);
        token = out[i];
    }
    fflush(stdout);
    if (verbose) {
        fprintf(stderr, "\n\n%d steps of %d beams in %.3f s\n", ran, n_beams, secs);
        for (int i = 0; i < n_beams; ++i)
            fprintf(stderr, "result %d: %d tokens, log-probability %g, normalised score %g\n", i, len[i], lp[i],
                    len[i] ? lp[i] / (float)len[i] : 0.0f);
    }
    return L2B_OK;
}

int main(int argc, char **argv) {
    if (argc < 2) { fputs(usage_text, stdout); return 0; }
    const char *bin_path = nullptr, *input = nullptr, *tokenizer_path = "tokenizer.bin";
    l2h_gen_options opt{1.0f, 0.9f, 0, 1, 0, 0, 0};
    int n_gpus = 1, draft_k = 3, n_beams = 0;
    const char *draft_path = nullptr;
    bool verbose = false;
    int32_t weight_format = L2B_WEIGHTS_F32, kv_flag = 0;
    l2h_seed((uint64_t)time(nullptr));
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        auto need = [&](const char *what) -> const char * {
            if (++i >= argc) { fprintf(stderr, "error: missing argument for %s\n", what); exit(1); }
            return argv[i];
        };
        if (a == "-h" || a == "--help") { fputs(usage_text, stdout); return 0; }
        else if (a[0] != '-') {
            if (bin_path) { fprintf(stderr, "error: multiple checkpoint paths specified\n"); return 1; }
            bin_path = argv[i];
        } else if (a == "-t" || a == "--temperature") opt.temperature = strtof(need("temperature"), nullptr);
        else if (a == "-n" || a == "--seq-len") opt.n_steps = atoi(need("seq-len"));
        else if (a == "-p" || a == "--top-p") { opt.top_p = strtof(need("top-p"), nullptr); if (opt.top_p < 0) opt.top_p = 0; if (opt.top_p > 1) opt.top_p = 1; }
        else if (a == "-i" || a == "--input") input = need("input");
        else if (a == "-z" || a == "--tokenizer") tokenizer_path = need("tokenizer");
        else if (a == "-s" || a == "--seed") l2h_seed(strtoull(need("seed"), nullptr, 10));
        else if (a == "-v" || a == "--verbose") verbose = true;
        else if (a == "--device-argmax") opt.use_device_argmax = 1;
        else if (a == "--device-sampler") opt.use_device_sampler = 1;
        else if (a == "--prefill") opt.use_prefill = 1;
        else if (a == "--gpus") n_gpus = atoi(need("gpus"));
        else if (a == "--draft") draft_path = need("draft");
        else if (a == "--draft-k") draft_k = atoi(need("draft-k"));
        else if (a == "--bf16") weight_format = L2B_WEIGHTS_BF16;
        else if (a == "--q8") weight_format = L2B_WEIGHTS_Q8;
        else if (a == "--kv-bf16") kv_flag = L2B_KV_BF16;
        else if (a == "--kv-e4m3") kv_flag = L2B_KV_E4M3;
        else if (a == "--beam") n_beams = atoi(need("beam"));
        else { fprintf(stderr, "error: unknown argument '%s'\n", argv[i]); fputs(usage_text, stdout); return 0; }
    }
    if (!bin_path) { fputs(usage_text, stdout); return 0; }
    if (n_beams && (n_beams < 1 || n_beams > L2B_BEAM_MAX || n_gpus != 1 || draft_path)) {
        fprintf(stderr, "error: --beam takes 1 to %d beams on one GPU, without --draft\n", L2B_BEAM_MAX);
        return 1;
    }

    l2h_checkpoint ck;
    if (l2h_load_checkpoint(bin_path, &ck) != L2B_OK) { fprintf(stderr, "error: cannot read checkpoint %s\n", bin_path); return 1; }
    const l2b_config &c = ck.config;
    if (verbose) {
        fprintf(stderr, "config: dim=%d hidden_dim=%d n_layers=%d n_heads=%d n_kv_heads=%d vocab_size=%d seq_len=%d\n",
                c.dim, c.hidden_dim, c.n_layers, c.n_heads, c.n_kv_heads, c.vocab_size, c.seq_len);
        fprintf(stderr, "shared weights: %s\ntemperature: %g\ntop-p: %g\n\n", c.shared_weights ? "true" : "false", opt.temperature, opt.top_p);
    }
    l2b_ctx *ctx = nullptr;
    const int32_t layout = n_beams ? L2B_KV_PAGED : 0;          // beam search needs the paged KV cache
    int32_t rc = l2b_create_format(&ctx, &c, ck.data, ck.n_floats, nullptr, nullptr, n_gpus, weight_format | kv_flag | layout);   // after :967
    if (rc) { fprintf(stderr, "error: l2b_create: %s (%s)\n", l2b_status_string(rc), l2b_last_error(nullptr)); return 1; }
    if (verbose) {
        int32_t fmt = 0;
        uint64_t n_rounded = 0;
        l2b_weight_info(ctx, &fmt, &n_rounded);
        fprintf(stderr, "weights: %s on the GPU, %llu matrix weights changed by rounding or quantization\n",
                fmt == L2B_WEIGHTS_BF16 ? "bf16" : fmt == L2B_WEIGHTS_Q8 ? "q8" : "fp32", (unsigned long long)n_rounded);
        print_kv_info("kv cache", ctx);
        fputc('\n', stderr);
    }
    l2h_free_checkpoint(&ck);   // host copy no longer needed: weights live in HBM
    l2b_ctx *draft = nullptr;
    l2b_config dc{};
    if (draft_path) {
        l2h_checkpoint dck;
        if (l2h_load_checkpoint(draft_path, &dck) != L2B_OK) { fprintf(stderr, "error: cannot read draft checkpoint %s\n", draft_path); return 1; }
        dc = dck.config;
        if (dc.vocab_size != c.vocab_size || dc.seq_len < c.seq_len) {
            fprintf(stderr, "error: the draft needs the target's vocab_size (%d) and a seq_len of at least %d\n", c.vocab_size, c.seq_len);
            return 1;
        }
        if (draft_k < 0 || draft_k > L2B_SPECULATIVE_MAX_K) { fprintf(stderr, "error: --draft-k must be in [0, %d]\n", L2B_SPECULATIVE_MAX_K); return 1; }
        rc = l2b_create_format(&draft, &dc, dck.data, dck.n_floats, nullptr, nullptr, 1, weight_format | kv_flag);
        if (rc) { fprintf(stderr, "error: l2b_create (draft): %s (%s)\n", l2b_status_string(rc), l2b_last_error(nullptr)); return 1; }
        if (verbose) print_kv_info("draft kv cache", draft);
        l2h_free_checkpoint(&dck);
    }

    l2h_tokenizer *tk = nullptr;
    if (l2h_tokenizer_load(tokenizer_path, c.vocab_size, &tk) != L2B_OK) { fprintf(stderr, "error: cannot read tokenizer %s\n", tokenizer_path); return 1; }
    std::vector<int32_t> prompt;
    if (input) {
        prompt.resize(strlen(input) + 1);
        const int32_t n = l2h_tokenizer_encode(tk, input, (int32_t)strlen(input), prompt.data(), (int32_t)prompt.size());
        if (n < 0) { fprintf(stderr, "error: cannot encode prompt\n"); return 1; }
        prompt.resize(n);
    }
    if (n_beams) {
        rc = generate_beam(ctx, c, n_beams, opt, prompt, tk, verbose);
        if (rc) { fprintf(stderr, "\nerror: %s (%s)\n", l2b_status_string(rc), l2b_last_error(ctx)); return 1; }
    } else if (draft) {
        rc = generate_with_draft(ctx, c, draft, dc, draft_k, opt, prompt, tk, verbose);
        if (rc) { fprintf(stderr, "\nerror: %s (%s / %s)\n", l2b_status_string(rc), l2b_last_error(ctx), l2b_last_error(draft)); return 1; }
    } else {
        l2h_gen_result res;
        rc = l2h_generate(ctx, &c, &opt, prompt.data(), (int32_t)prompt.size(), tk, nullptr, 0, &res);
        if (rc) { fprintf(stderr, "\nerror: %s (%s)\n", l2b_status_string(rc), l2b_last_error(ctx)); return 1; }
        if (verbose && res.secs_after_first > 0)   // :1043-1050: (pos - 1) / elapsed since the first token
            fprintf(stderr, "\n\n%d tokens per second\n", (int)((res.n_forward - 1) / res.secs_after_first));
    }
    l2h_tokenizer_free(tk);
    l2b_destroy(draft);
    l2b_destroy(ctx);
    return 0;
}
