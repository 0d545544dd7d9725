// llama2_b200 — command-line twin of the reference's `llama2` binary (src/main.zig:823-1051)
// with transformer() served by the H100 library.  Same flags and usage text (:800-813).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

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
    "     --gpus <1|2|4|8>      tensor-parallel over that many GPUs (llama2-7B class models)\n";

int main(int argc, char **argv) {
    if (argc < 2) { fputs(usage_text, stdout); return 0; }
    const char *bin_path = nullptr, *input = nullptr, *tokenizer_path = "tokenizer.bin";
    l2h_gen_options opt{1.0f, 0.9f, 0, 1, 0, 0, 0};
    int n_gpus = 1;
    bool verbose = false;
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
        else { fprintf(stderr, "error: unknown argument '%s'\n", argv[i]); fputs(usage_text, stdout); return 0; }
    }
    if (!bin_path) { fputs(usage_text, stdout); return 0; }

    l2h_checkpoint ck;
    if (l2h_load_checkpoint(bin_path, &ck) != L2B_OK) { fprintf(stderr, "error: cannot read checkpoint %s\n", bin_path); return 1; }
    const l2b_config &c = ck.config;
    if (verbose) {
        fprintf(stderr, "config: dim=%d hidden_dim=%d n_layers=%d n_heads=%d n_kv_heads=%d vocab_size=%d seq_len=%d\n",
                c.dim, c.hidden_dim, c.n_layers, c.n_heads, c.n_kv_heads, c.vocab_size, c.seq_len);
        fprintf(stderr, "shared weights: %s\ntemperature: %g\ntop-p: %g\n\n", c.shared_weights ? "true" : "false", opt.temperature, opt.top_p);
    }
    l2b_ctx *ctx = nullptr;
    int32_t rc = l2b_create(&ctx, &c, ck.data, ck.n_floats, nullptr, nullptr, n_gpus);   // after :967
    if (rc) { fprintf(stderr, "error: l2b_create: %s (%s)\n", l2b_status_string(rc), l2b_last_error(nullptr)); return 1; }
    l2h_free_checkpoint(&ck);   // host copy no longer needed: weights live in HBM

    l2h_tokenizer *tk = nullptr;
    if (l2h_tokenizer_load(tokenizer_path, c.vocab_size, &tk) != L2B_OK) { fprintf(stderr, "error: cannot read tokenizer %s\n", tokenizer_path); return 1; }
    std::vector<int32_t> prompt;
    if (input) {
        prompt.resize(strlen(input) + 1);
        const int32_t n = l2h_tokenizer_encode(tk, input, (int32_t)strlen(input), prompt.data(), (int32_t)prompt.size());
        if (n < 0) { fprintf(stderr, "error: cannot encode prompt\n"); return 1; }
        prompt.resize(n);
    }
    l2h_gen_result res;
    rc = l2h_generate(ctx, &c, &opt, prompt.data(), (int32_t)prompt.size(), tk, nullptr, 0, &res);
    if (rc) { fprintf(stderr, "\nerror: %s (%s)\n", l2b_status_string(rc), l2b_last_error(ctx)); return 1; }
    if (verbose && res.secs_after_first > 0)   // :1043-1050: (pos - 1) / elapsed since the first token
        fprintf(stderr, "\n\n%d tokens per second\n", (int)((res.n_forward - 1) / res.secs_after_first));
    l2h_tokenizer_free(tk);
    l2b_destroy(ctx);
    return 0;
}
