// llama2_b200.cu — C ABI (include/llama2_b200.h) over the sm_90a kernels in l2b_device.cuh.
//
// Replaces transformer() of the reference (src/main.zig:285-430) and the device-side
// equivalents of Weights.init (:73-115) / RunState.init (:137-154).  Pure CUDA runtime:
// no torch, no CPU fallback.  One rank = one GPU = one stream; a decode step is a CUDA graph
// of 5 kernels per layer + classifier, replayed per token.  A context is either one rank
// (single GPU, or one process per GPU with peers reached through CUDA IPC) or a group of ranks
// inside one process (l2b_create with n_gpus > 1: peers reached through UVA peer access).
#include "../../include/llama2_b200.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <chrono>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

#include "l2b_device.cuh"

using namespace l2b;

// ---------------------------------------------------------------------------------------
// NCCL through dlopen: single-GPU use never needs libnccl (or its headers) to be present.  NCCL
// is only the bootstrap of the one-process-per-GPU mode (it carries the CUDA IPC handles at
// create time) and the data plane of the L2B_TP=nccl baseline; the default data plane is this
// library's own peer-memory exchange.  The few types / enum values used are restated here.
// ---------------------------------------------------------------------------------------
namespace {
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
constexpr int ncclSuccess = 0;
constexpr int ncclChar = 0, ncclInt = 2, ncclUint64 = 5, ncclFloat = 7;   // ncclDataType_t
constexpr int ncclSum = 0, ncclMax = 2;                                   // ncclRedOp_t

struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};
NcclApi g_nccl;

bool nccl_load(std::string *err) {
    if (g_nccl.ok) return true;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *n : names) {
        g_nccl.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_nccl.handle) break;
    }
    if (!g_nccl.handle) {
        if (err) *err = std::string("dlopen(libnccl.so.2) failed: ") + dlerror();
        return false;
    }
#define L2B_SYM(field, name)                                                        \
    *(void **)(&g_nccl.field) = dlsym(g_nccl.handle, name);                         \
    if (!g_nccl.field) {                                                            \
        if (err) *err = std::string("dlsym failed: ") + name;                       \
        return false;                                                               \
    }
    L2B_SYM(GetUniqueId, "ncclGetUniqueId");
    L2B_SYM(CommInitRank, "ncclCommInitRank");
    L2B_SYM(CommDestroy, "ncclCommDestroy");
    L2B_SYM(AllReduce, "ncclAllReduce");
    L2B_SYM(AllGather, "ncclAllGather");
    L2B_SYM(GetErrorString, "ncclGetErrorString");
#undef L2B_SYM
    g_nccl.ok = true;
    return true;
}
}  // namespace

// ---------------------------------------------------------------------------------------
// Context (one rank)
// ---------------------------------------------------------------------------------------
enum StepMode { MODE_LOGITS = 0, MODE_ARGMAX = 1, MODE_SAMPLE = 2, MODE_NOCLS = 3 };
enum GraphId { G_LOGITS = 0, G_ARGMAX_ONE = 1, G_ARGMAX_LOOP = 2, G_SAMPLE = 3, G_PREFILL_LOOP = 4, G_SCORE_LOOP = 5,
               G_COUNT = 6 };
constexpr int kCandCap = 8192;               // top-p candidates returned per step (more => host filters itself)

// The device weights and RoPE tables of one loaded model (one rank's shard), shared by the context that
// loaded them and every session created on it (l2b_create_session); freed with the last of them.
// The KV pages of a paged model (L2B_KV_PAGED): [L][K rows P | V rows P][kv_loc] elements each, P =
// KV_PAGE_ROWS.  Released pages go to the free list, not to the device, and are not cleared: no kernel reads
// a row past its stream's end.  The null page is what every unassigned page-table entry points at, so
// the rows a kernel loads and then masks (split 0's first pass) are always valid memory.
struct KvPool {
    size_t page_bytes = 0;
    void *null_page = nullptr;
    std::vector<void *> all;                  // every page allocated, freed with the model
    std::vector<void *> free_pages;
    std::unordered_map<void *, int> refs;     // pages in use -> how many sessions hold them
    uint64_t limit = 0;                       // l2b_kv_pool_limit (0: none)
};

struct SharedWeights {
    int refs = 1;
    std::vector<void *> owned;
    KvPool *pool = nullptr;                   // paged models only
    // e4m3 KV formats only: [L][s_k, s_v] (l2b_kv_scales) on the device, read by the kernels through a
    // pointer so captured graphs stay valid, and its host copy (l2b_read_state's widening)
    float *kv_scale = nullptr;
    std::vector<float> kv_scale_h;
};

struct l2b_ctx {
    l2b_config cfg{};
    int rank = 0, world = 1, device = 0, num_sms = 0;
    // in-process group (l2b_create with n_gpus > 1): the leader (rank 0) owns the other ranks
    std::vector<l2b_ctx *> members;          // leader only: all ranks, [0] == this
    l2b_ctx *leader = nullptr;
    // derived sizes (local = this rank's shard)
    int dim = 0, hidden = 0, head_size = 0, kv_mul = 0;
    int q_dim = 0, kv_dim = 0;              // global
    int q_loc = 0, kv_loc = 0, hid_loc = 0, heads_loc = 0, vocab_loc = 0;
    // device weights (Weights, src/main.zig:53-71), this rank's slices, owned by `weights`
    SharedWeights *weights = nullptr;
    float *rms_att = nullptr, *rms_ffn = nullptr, *rms_final = nullptr;
    // matrix weights in the device format `wfmt` (l2b_weight_format): fp32, bf16 with rows padded to
    // w_pitch<bf16>(cols) elements, or q8 row records of w_pitch<q8>(cols) bytes; address them with wrow()
    int wfmt = L2B_WEIGHTS_F32;
    uint64_t n_rounded = 0;                  // matrix weights the bf16 rounding / q8 quantization changed (l2b_weight_info)
    unsigned long long *d_rounded = nullptr; // ... counted on the device while synthetic weights are generated
    void *emb = nullptr;
    void *wq = nullptr, *wk = nullptr, *wv = nullptr, *wo = nullptr;
    void *w1 = nullptr, *w2 = nullptr, *w3 = nullptr, *wcls = nullptr;
    // device run state (RunState, :119-135)
    float *X = nullptr;                      // residual stream x; wo / w2 add into it (:395, :422)
    float *Xalt = nullptr;                   // second copy: kernels that fold partial vectors in write the new x here (ping-pong)
    float *final_X = nullptr;                // which of the two holds x after a step
    float *attn_parts = nullptr;             // small-model fusion: (n_heads, dim) partial vectors of attention + wo
    bool fuse_attn = false;
    // batched prompt prefill (l2b_prefill) and batched step (l2b_forward_batch) on bandwidth-bound shapes:
    // PF_MAXB vectors per weight pass
    float *pf_x = nullptr, *pf_q = nullptr, *pf_xb = nullptr, *pf_hb = nullptr;   // [PF_MAXB][dim | q | q | hidden]
    float *pf_logits = nullptr;                                                  // [PF_MAXB][vocab]
    unsigned long long *pf_amax = nullptr;                                       // [PF_MAXB] packed argmax keys
    float *pf_part_o = nullptr, *pf_part_ml = nullptr;
    unsigned int *pf_counters = nullptr;
    bool pf_ready = false, pf_ok = false;
    int *call_ints = nullptr;                // a batched call's tokens and other per-call ints (batched_begin),
    size_t call_ints_cap = 0;                // grown on demand
    ProbIndex *call_cand = nullptr;          // l2b_verify_sample_ragged: kCandCap candidates per position,
    size_t call_cand_cap = 0;                // grown on demand
    unsigned char *h_call = nullptr;         // ... and its pinned D2H staging (probabilities, candidates)
    size_t h_call_bytes = 0;
    float *delta = nullptr;                  // L2B_TP=nccl baseline only: partial rows before the NCCL all-reduce
    float *q = nullptr, *xb = nullptr, *hb = nullptr, *logits = nullptr, *logits_loc = nullptr;
    // KV cache, (L, seq_len, kv_loc) elements of the format `kvfmt`: 0 (fp32), L2B_KV_BF16, L2B_KV_E4M3,
    // or L2B_KV_ROUND_BF16 / L2B_KV_ROUND_E4M3 (fp32 elements holding rounded values: the references)
    int kvfmt = 0;
    void *kcache = nullptr, *vcache = nullptr;
    // Paged layout (L2B_KV_PAGED): kcache and vcache are both the device page table kv_tab, [L][n_pages]
    // addresses of layer l's K row jP in page j (its V rows follow P rows later); pages[j] is the page
    // this session holds for positions [jP, jP+P), or nullptr (the table entry points at the null page).
    // h_tab is the table's pinned host mirror; the device copy never moves, so captured graphs stay valid.
    bool paged = false;
    int n_pages = 0;
    std::vector<void *> pages;
    void **kv_tab = nullptr, **h_tab = nullptr;
    bool tab_dirty = false;                  // h_tab has entries the device table does not
    float *rope_cos = nullptr, *rope_sin = nullptr; // (seq_len, head_size/2)
    float *part_o = nullptr, *part_ml = nullptr;
    unsigned int *counters = nullptr;
    int *ctl = nullptr;
    unsigned long long *amax = nullptr;
    int *gen_forced = nullptr, *gen_out = nullptr, *gen_ndone = nullptr;
    ProbIndex *cand = nullptr;               // sampler: top-p candidates (index order)
    int *n_cand = nullptr;
    float *score_lp = nullptr;               // l2b_score: seq_len log-probabilities and greedy tokens
    int *score_greedy = nullptr;
    // host pinned
    float *h_logits = nullptr;               // vocab floats: logits, or probabilities after sample_prep
    int *h_ctl = nullptr;                    // [0..7] host -> device control words, [8..15] device -> host status
    int *h_ints = nullptr;                   // [0]=next, [1]=n_done, [2]=n_cand
    int *h_gen = nullptr;                    // seq_len ints
    ProbIndex *h_cand = nullptr;
    // attention launch shape
    int nsplit = 1, min_chunk = 256, attn_smem = 0;   // timeline splits of >= 256 positions
    int attn_pg_bytes = 0, attn_pg_bytes_wo = 0;      // paged: shared memory for a split's page addresses
    // streams / graphs
    cudaStream_t stream = nullptr;
    cudaGraphExec_t graphs[G_COUNT] = {};
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool use_graphs = true;
    bool use_pdl = true;
    bool time_steps = false;                 // L2B_TIME_STEPS=1: CUDA events around every single step (l2b_last_timing)
    int last_grid = 0;                       // grid of the most recent GEMV launch
    // tensor-parallel exchange over peer memory (world > 1).  One arena per rank holds every landing
    // area, so one IPC handle (or one UVA pointer) per rank is all the ranks trade at create time:
    //   ll_red    [2L reduce points][world source ranks][dim] LL units   (wo / w2 partial rows)
    //   ll_logits [vocab] LL units                                       (classifier slices of all ranks)
    //   ll_amax   [world][2] LL units                                    (packed argmax keys)
    bool use_p2p = false;
    unsigned char *arena = nullptr;
    size_t arena_bytes = 0, off_red = 0, off_logits = 0, off_amax = 0;
    unsigned char *peer_arena[MAX_TP] = {};
    std::vector<void *> ipc_opened;
    unsigned long long spin_ns = 20ull * 1000000000ull;   // bound on every peer wait (L2B_SPIN_TIMEOUT_MS)
    bool attn_flash = true;                  // flash-decoding attention (false: 3-pass kernel)
    unsigned long long *trace = nullptr;     // L2B_TRACE=1: [launch][TRACE_MAX_CTAS][TRACE_SLOTS] timeline
    int trace_launches = 0;
    int tma_stages = 0;                      // 0 = auto; else forced ring depth
    int tma_prefill = 0;                     // stages in flight before the dependency wait; 0 = the whole ring (L2B_TMA_PREFILL)
    bool big_kernel_tma = true;              // bandwidth-bound GEMVs: TMA-ring kernel (false: register-fed 8-row kernel)
    long long gemv8_min_bytes = 8ll << 20;   // >= this many weight bytes (and n >= big_min_n): streaming kernel; -1 = never
    int big_min_n = 1024;                    // measured r02: at n = 768 the TMA ring (192 of 256 columns per stage) loses to the latency kernel
    int force_kernel = 0;                    // l2b_op_fused_matmul: 0 auto, 1 small, 2 register-fed 8-row, 3 TMA ring
    int launches_per_step = 0;
    std::set<const void *> attr_done;        // kernels whose max-dynamic-smem attribute is set on this device
    // comm (bootstrap / nccl baseline)
    ncclComm_t comm = nullptr;
    // bookkeeping
    int n_appended = 0;
    float last_ms = 0.0f;
    int last_launches = 0;
    double load_ms = 0.0;                    // checkpoint upload wall time (l2b_load_stats)
    uint64_t load_bytes = 0;
    std::string err;
    std::vector<void *> owned;              // device allocations to free
    // upload staging (pinned, double-buffered)
    unsigned char *stage[2] = {nullptr, nullptr};
    cudaEvent_t stage_ev[2] = {nullptr, nullptr};
    size_t stage_bytes = 0;
    int stage_next = 0;
    // per-kernel profiling (l2b_profile_step)
    bool profiling = false;
    std::vector<cudaEvent_t> prof_ev;
    std::vector<l2b_kernel_time> prof_rec;
};

namespace {

const char *kNoError = "";
thread_local std::string g_create_error;

#define L2B_CUDA(ctx, call)                                                                   \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            char buf__[512];                                                                  \
            snprintf(buf__, sizeof buf__, "%s failed: %s (%s:%d)", #call,                     \
                     cudaGetErrorString(e__), __FILE__, __LINE__);                            \
            (ctx)->err = buf__;                                                               \
            return (e__ == cudaErrorMemoryAllocation) ? L2B_ERR_OOM : L2B_ERR_CUDA;           \
        }                                                                                     \
    } while (0)

#define L2B_NCCL(ctx, call)                                                                   \
    do {                                                                                      \
        ncclResult_t r__ = (call);                                                            \
        if (r__ != ncclSuccess) {                                                             \
            char buf__[512];                                                                  \
            snprintf(buf__, sizeof buf__, "%s failed: %s (%s:%d)", #call,                     \
                     g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "?", __FILE__,      \
                     __LINE__);                                                               \
            (ctx)->err = buf__;                                                               \
            return L2B_ERR_COMM;                                                              \
        }                                                                                     \
    } while (0)

int fail(l2b_ctx *ctx, int code, const char *msg) {
    if (ctx) ctx->err = msg;
    return code;
}

// all ranks this handle drives from this process (1 unless it is an in-process group)
std::vector<l2b_ctx *> locals(l2b_ctx *ctx) {
    if (!ctx->members.empty()) return ctx->members;
    return std::vector<l2b_ctx *>{ctx};
}

// a device allocation freed with the context, or with the model's weights when owner is given
template <typename T>
int dev_alloc(l2b_ctx *ctx, T **p, size_t count, std::vector<void *> *owner = nullptr) {
    void *q = nullptr;
    L2B_CUDA(ctx, cudaMalloc(&q, (count ? count : 1) * sizeof(T)));
    (owner ? owner : &ctx->owned)->push_back(q);
    *p = static_cast<T *>(q);
    return L2B_OK;
}

// ---- formats: the one place a weight or KV format value becomes the C++ type the kernels are templated on.
// Each visitor calls f(type_tag<T>()) and has a case for every format; split_format admits no other value,
// so anything else is a defect here and aborts.
template <typename T> struct type_tag { typedef T type; };

// ---- device weight format: the weight element W (float, bf16 or q8)
template <typename F>
auto with_w(int wfmt, F f) {
    switch (wfmt) {
    case L2B_WEIGHTS_F32: return f(type_tag<float>());
    case L2B_WEIGHTS_BF16: return f(type_tag<bf16>());
    case L2B_WEIGHTS_Q8: return f(type_tag<q8>());
    }
    abort();
}
// bytes of a stored element and elements from one row to the next, of a matrix in the context's format
size_t w_elem(const l2b_ctx *ctx) { return with_w(ctx->wfmt, [](auto w) { return sizeof(typename decltype(w)::type); }); }
uint64_t w_ld(const l2b_ctx *ctx, uint64_t cols) {
    return with_w(ctx->wfmt, [cols](auto w) { return (uint64_t)w_pitch<typename decltype(w)::type>((int)cols); });
}

// ---- KV-cache format (kvfmt, with the layout flag `paged` apart)
// the element E a cache stores: the round-trip references are fp32 caches
template <typename F>
auto with_kv_elem(int kvfmt, F f) {
    switch (kvfmt) {
    case 0:                                       // fp32
    case L2B_KV_ROUND_BF16:
    case L2B_KV_ROUND_E4M3: return f(type_tag<float>());
    case L2B_KV_BF16: return f(type_tag<bf16>());
    case L2B_KV_E4M3: return f(type_tag<e4m3>());
    }
    abort();
}
// f(type_tag<E>()) or f(type_tag<kv_paged<E>>()) for element type E
template <typename E, typename F>
auto kv_layout(bool paged, F f) { return paged ? f(type_tag<kv_paged<E>>()) : f(type_tag<E>()); }
// the KV type the QKV epilogue writes the context's cache with: float, bf16, kv_f32_bf16, e4m3 or kv_f32_e4m3,
// in its kv_paged<> form on a paged cache
template <typename F>
auto with_kv_store(const l2b_ctx *ctx, F f) {
    switch (ctx->kvfmt) {
    case 0: return kv_layout<float>(ctx->paged, f);
    case L2B_KV_BF16: return kv_layout<bf16>(ctx->paged, f);
    case L2B_KV_ROUND_BF16: return kv_layout<kv_f32_bf16>(ctx->paged, f);
    case L2B_KV_E4M3: return kv_layout<e4m3>(ctx->paged, f);
    case L2B_KV_ROUND_E4M3: return kv_layout<kv_f32_e4m3>(ctx->paged, f);
    }
    abort();
}
// the KV type the attention kernels read the context's cache with: its element, kv_paged<> on a paged cache
template <typename F>
auto with_kv_read(const l2b_ctx *ctx, F f) {
    return with_kv_elem(ctx->kvfmt, [ctx, &f](auto e) { return kv_layout<typename decltype(e)::type>(ctx->paged, f); });
}
size_t kv_elem(const l2b_ctx *ctx) { return with_kv_elem(ctx->kvfmt, [](auto e) { return sizeof(typename decltype(e)::type); }); }
// n stored elements at `from` widened on the host to the fp32 values they stand for (e4m3: under the layer's
// scale s).  Front to back, each element read before its value is written, so `to` may overlap `from` where
// value i ends at or below element i + 1 (the in-place widening of l2b_read_state).
void kv_widen(type_tag<float>, const unsigned char *from, float *to, uint64_t n, float) { memmove(to, from, n * 4); }
void kv_widen(type_tag<bf16>, const unsigned char *from, float *to, uint64_t n, float) {
    for (uint64_t i = 0; i < n; ++i) {
        uint16_t h;
        memcpy(&h, from + 2 * i, 2);
        const uint32_t u = (uint32_t)h << 16;
        memcpy(to + i, &u, 4);
    }
}
void kv_widen(type_tag<e4m3>, const unsigned char *from, float *to, uint64_t n, float s) {
    for (uint64_t i = 0; i < n; ++i) to[i] = e4m3_widen(from[i], s);
}
// the formats whose kernels take the model's scales: the e4m3 cache and its fp32 reference
bool kv_scaled(int kvfmt) { return kvfmt == L2B_KV_E4M3 || kvfmt == L2B_KV_ROUND_E4M3; }
// layer l's (s_k, s_v) on the device, or nullptr for a format without scales
const float *kv_scale_at(const l2b_ctx *ctx, int l) {
    return ctx->weights && ctx->weights->kv_scale ? ctx->weights->kv_scale + 2 * (size_t)l : nullptr;
}
// layer `layer` of a cache (kcache or vcache) of ctx: its base, or (paged) its page table
void *kv_layer(const l2b_ctx *ctx, void *cache, int layer) {
    if (ctx->paged) return static_cast<void **>(cache) + (size_t)layer * ctx->n_pages;
    return static_cast<unsigned char *>(cache) + (size_t)layer * ctx->cfg.seq_len * ctx->kv_loc * kv_elem(ctx);   // :354
}
// row `row` of a matrix of `cols` columns that starts at base
const void *wrow(const l2b_ctx *ctx, const void *base, uint64_t row, uint64_t cols) {
    return static_cast<const unsigned char *>(base) + row * w_ld(ctx, cols) * w_elem(ctx);
}

// ---- shape validation (the reference's asserts, src/main.zig:433-434,:534-540,:658-661) ----
int validate_config(const l2b_config *c, int world, std::string *why) {
    auto bad = [&](const char *m) { *why = m; return L2B_ERR_UNSUPPORTED; };
    if (c->dim <= 0 || c->hidden_dim <= 0 || c->n_layers <= 0 || c->n_heads <= 0 ||
        c->n_kv_heads <= 0 || c->vocab_size <= 0 || c->seq_len <= 0) {
        *why = "config fields must be positive";
        return L2B_ERR_INVALID_ARG;
    }
    if (c->dim % c->n_heads) return bad("dim % n_heads != 0");
    if (c->n_heads % c->n_kv_heads) return bad("n_heads % n_kv_heads != 0");
    const int hs = c->dim / c->n_heads;
    if (c->dim % 4 || c->hidden_dim % 4) return bad("dim and hidden_dim must be multiples of 4");
    if (hs % 4) return bad("head_size must be a multiple of 4");
    // the attention kernels write one output element per thread (NT = 256) and the RoPE row of a
    // position is staged as head_size/2 <= 128 pairs
    if (hs > NT) return bad("head_size > 256 is not supported");
    if (world != 1 && world != 2 && world != 4 && world != 8) return bad("world_size must be 1, 2, 4 or 8");
    if (c->n_kv_heads % world) return bad("n_kv_heads % world_size != 0");
    if ((c->hidden_dim / world) % 4 || c->hidden_dim % world) return bad("hidden_dim/world_size must be a multiple of 4");
    if (c->vocab_size % world || (world > 1 && (c->vocab_size / world) % 2)) return bad("vocab_size/world_size must be an even integer");
    return L2B_OK;
}

uint64_t checkpoint_floats(const l2b_config *c) {
    const uint64_t dim = c->dim, hid = c->hidden_dim, L = c->n_layers, V = c->vocab_size, S = c->seq_len;
    const uint64_t hs = dim / c->n_heads, kvd = hs * c->n_kv_heads;
    uint64_t n = V * dim + L * dim + L * dim * dim + 2 * L * dim * kvd + L * dim * dim + L * dim +
                 3 * L * dim * hid + dim + 2 * (S * hs / 2);
    if (!c->shared_weights) n += V * dim;
    return n;
}

// ---- tensor materialisation: upload a (possibly sharded) window, or synthesise it in place ----
enum ShardMode { SH_NONE, SH_ROWS, SH_COLS };
struct Dist { double mean, sigma; float lo, hi; };
constexpr double kSynthInvStd = 2.6428997921303014e-05;  // 1 / sqrt(4*(65536^2-1)/12)

struct Source {
    const float *host = nullptr;   // checkpoint payload or nullptr => synthetic
    uint64_t seed = 0;
};

// Checkpoint ingest (SURVEY 8f.3; the reference slurps the file into pageable heap memory,
// src/main.zig:955-964).  The caller's buffer is pageable, so a plain cudaMemcpy would bounce every
// byte through the driver's small internal staging buffer synchronously.  Here the payload moves
// in chunks through two pinned buffers: while chunk k is in flight on the copy engine, the host
// is already filling the other buffer with chunk k+1 (for column-sharded tensors the host-side
// fill also compacts the strided window, so the DMA is always a dense 1-D copy).
// Quantizes one row of cols fp32 weights into a q8 row record (w_pitch<q8>(cols) bytes, padding zeroed);
// returns how many weights the quantization changed, or -1 when the row holds a non-finite value.
int64_t quantize_q8_row(const float *w, uint64_t cols, unsigned char *rec) {
    const int ng = q8_groups((int)cols), so = q8_scale_off((int)cols);
    float *scales = reinterpret_cast<float *>(rec + so);
    memset(rec, 0, (size_t)w_pitch<q8>((int)cols));
    int64_t changed = 0;
    for (int g = 0; g < ng; ++g) {
        const uint64_t c0 = (uint64_t)g * Q8_GROUP, c1 = std::min<uint64_t>(cols, c0 + Q8_GROUP);
        float a = 0.0f;
        for (uint64_t c = c0; c < c1; ++c) {
            if (!std::isfinite(w[c])) return -1;
            a = std::max(a, std::fabs(w[c]));
        }
        const float s = q8_scale(a);
        for (uint64_t c = c0; c < c1; ++c) {
            const int8_t q = q8_code(w[c], a, s);
            const float d = q8_dequant(q, s);
            changed += memcmp(&d, w + c, 4) != 0;
            rec[c] = (unsigned char)q;
        }
        memcpy(scales + g, &s, 4);
    }
    return changed;
}

// Rounds one row of cols fp32 weights to bf16 (bf16_round_bits) into d, zero-padded to ld elements; returns
// how many weights the rounding changed.
int64_t round_bf16_row(const float *w, uint64_t cols, uint64_t ld, uint16_t *d) {
    int64_t changed = 0;
    for (uint64_t c = 0; c < cols; ++c) {
        uint32_t u;
        memcpy(&u, w + c, 4);
        d[c] = bf16_round_bits(u);
        changed += ((uint32_t)d[c] << 16) != u;
    }
    for (uint64_t c = cols; c < ld; ++c) d[c] = 0;
    return changed;
}

template <typename W>
int upload(l2b_ctx *ctx, void *dst, const float *src, uint64_t rows, uint64_t cols, uint64_t src_pitch) {
    if (!ctx->stage[0]) {
        size_t want = 32ull << 20;
        const char *env = getenv("L2B_STAGE_MB");
        if (env && atoi(env) > 0) want = (size_t)atoi(env) << 20;
        ctx->stage_bytes = want;
        for (int i = 0; i < 2; ++i) {
            L2B_CUDA(ctx, cudaHostAlloc((void **)&ctx->stage[i], want, cudaHostAllocDefault));
            L2B_CUDA(ctx, cudaEventCreateWithFlags(&ctx->stage_ev[i], cudaEventDisableTiming));
        }
    }
    // Each row is packed into the stage in its stored form, so the DMA moves dense rows: bf16 rows are
    // rounded and padded with zeros to w_pitch elements (round_bf16_row), q8 rows quantized into their row
    // records (quantize_q8_row).
    const uint64_t ld = (uint64_t)w_pitch<W>((int)cols);
    const uint64_t row_bytes = ld * sizeof(W);
    const bool dense = (src_pitch == cols) && std::is_same<W, float>::value;
    const uint64_t total = rows * row_bytes;
    uint64_t done = 0;                       // bytes of the dense destination already issued
    while (done < total) {
        const int b = ctx->stage_next;
        ctx->stage_next ^= 1;
        L2B_CUDA(ctx, cudaEventSynchronize(ctx->stage_ev[b]));   // previous DMA out of this buffer finished
        uint64_t chunk = total - done < ctx->stage_bytes ? total - done : ctx->stage_bytes;
        if (dense) {
            memcpy(ctx->stage[b], reinterpret_cast<const unsigned char *>(src) + done, chunk);
        } else {
            // whole rows only (a chunk never splits a row of a sharded window)
            const uint64_t r = chunk / row_bytes;
            if (r == 0) return fail(ctx, L2B_ERR_UNSUPPORTED, "row larger than the upload staging buffer");
            chunk = r * row_bytes;
            const uint64_t row0 = done / row_bytes;
            for (uint64_t i = 0; i < r; ++i) {
                const float *s = src + (row0 + i) * src_pitch;
                unsigned char *d = ctx->stage[b] + i * row_bytes;
                int64_t changed = 0;
                if constexpr (std::is_same<W, q8>::value) {
                    changed = quantize_q8_row(s, cols, d);
                    if (changed < 0) return fail(ctx, L2B_ERR_INVALID_ARG, "non-finite matrix weight in a q8 payload");
                } else if constexpr (std::is_same<W, bf16>::value) {
                    changed = round_bf16_row(s, cols, ld, reinterpret_cast<uint16_t *>(d));
                } else {
                    static_assert(std::is_same<W, float>::value, "a weight element type");
                    memcpy(d, s, row_bytes);
                }
                ctx->n_rounded += (uint64_t)changed;
            }
        }
        L2B_CUDA(ctx, cudaMemcpyAsync(reinterpret_cast<unsigned char *>(dst) + done, ctx->stage[b], chunk,
                                      cudaMemcpyHostToDevice, ctx->stream));
        L2B_CUDA(ctx, cudaEventRecord(ctx->stage_ev[b], ctx->stream));
        done += chunk;
    }
    ctx->load_bytes += total;
    return L2B_OK;
}

// A tensor stored as elements W.  A bf16 or q8 matrix is only ever whole (single GPU).
template <typename W>
int materialize(l2b_ctx *ctx, void **dptr, const Source &src, uint64_t payload_off, int tensor_id,
                uint64_t L, uint64_t rows, uint64_t cols, ShardMode mode, Dist dist) {
    const uint64_t g = ctx->world, r = ctx->rank;
    const uint64_t rows_loc = (mode == SH_ROWS) ? rows / g : rows;
    const uint64_t cols_loc = (mode == SH_COLS) ? cols / g : cols;
    const uint64_t row0 = (mode == SH_ROWS) ? r * rows_loc : 0;
    const uint64_t col0 = (mode == SH_COLS) ? r * cols_loc : 0;
    const uint64_t ld = (uint64_t)w_pitch<W>((int)cols_loc);
    const size_t esize = sizeof(W);
    constexpr bool f32 = std::is_same<W, float>::value;
    unsigned char *base = nullptr;
    int rc = dev_alloc(ctx, &base, L * rows_loc * ld * esize, &ctx->weights->owned);
    if (rc) return rc;
    *dptr = base;
    const uint64_t tensor_seed = mix64(src.seed * 1000003ull + (uint64_t)tensor_id);
    const bool whole = (rows_loc == rows && cols_loc == cols);
    const uint64_t nl = whole ? 1 : L;            // one shot when nothing is cut
    const uint64_t rr = whole ? L * rows : rows_loc;
    if (!f32 && !src.host) {
        // the row padding (the upload writes its own zeros), and the device count of weights the synthesis
        // rounds, read back when the weights are in place
        L2B_CUDA(ctx, cudaMemsetAsync(base, 0, L * rows_loc * ld * esize, ctx->stream));
        if (!ctx->d_rounded) {
            if ((rc = dev_alloc(ctx, &ctx->d_rounded, 1))) return rc;
            L2B_CUDA(ctx, cudaMemsetAsync(ctx->d_rounded, 0, sizeof(unsigned long long), ctx->stream));
        }
    }
    for (uint64_t l = 0; l < nl; ++l) {
        void *dst = base + l * rows_loc * ld * esize;
        const uint64_t first = l * rows * cols + row0 * cols + col0;
        if (src.host) {
            rc = upload<W>(ctx, dst, src.host + payload_off + first, rr, cols_loc, cols);
            if (rc) return rc;
        } else {
            const uint64_t total = rr * cols_loc;
            int blocks = (int)((total + 255) / 256 < (uint64_t)(ctx->num_sms * 16)
                                   ? (total + 255) / 256
                                   : (uint64_t)(ctx->num_sms * 16));
            if (blocks < 1) blocks = 1;
            if constexpr (std::is_same<W, q8>::value) {
                const uint64_t groups = rr * (uint64_t)q8_groups((int)cols_loc);   // one thread per group
                const int gblocks = (int)std::min<uint64_t>((groups + 255) / 256, (uint64_t)ctx->num_sms * 16);
                synth_fill_q8_kernel<<<gblocks < 1 ? 1 : gblocks, 256, 0, ctx->stream>>>(
                    static_cast<unsigned char *>(dst), rr, cols_loc, first, cols, tensor_seed, dist.mean,
                    dist.sigma * kSynthInvStd, dist.lo, dist.hi, ctx->d_rounded);
            } else if constexpr (std::is_same<W, bf16>::value) {
                synth_fill_bf16_kernel<<<blocks, 256, 0, ctx->stream>>>(
                    static_cast<uint16_t *>(dst), rr, cols_loc, first, cols, tensor_seed, dist.mean,
                    dist.sigma * kSynthInvStd, dist.lo, dist.hi, ctx->d_rounded);
            } else {
                static_assert(f32, "a weight element type");
                synth_fill_kernel<<<blocks, 256, 0, ctx->stream>>>(static_cast<float *>(dst), rr, cols_loc, first, cols,
                                                                   tensor_seed, dist.mean, dist.sigma * kSynthInvStd,
                                                                   dist.lo, dist.hi);
            }
            L2B_CUDA(ctx, cudaGetLastError());
        }
    }
    return L2B_OK;
}
// matrix: a weight matrix, stored in the context's format (wfmt); otherwise fp32 (RMSNorm gains)
int materialize(l2b_ctx *ctx, void **dptr, const Source &src, uint64_t payload_off, int tensor_id,
                uint64_t L, uint64_t rows, uint64_t cols, ShardMode mode, Dist dist, bool matrix) {
    auto as = [&](auto w) { return materialize<typename decltype(w)::type>(ctx, dptr, src, payload_off, tensor_id, L, rows, cols, mode, dist); };
    return matrix ? with_w(ctx->wfmt, as) : as(type_tag<float>());
}
int materialize(l2b_ctx *ctx, float **dptr, const Source &src, uint64_t payload_off, int tensor_id,
                uint64_t L, uint64_t rows, uint64_t cols, ShardMode mode, Dist dist) {
    void *p = nullptr;
    const int rc = materialize(ctx, &p, src, payload_off, tensor_id, L, rows, cols, mode, dist, false);
    *dptr = static_cast<float *>(p);
    return rc;
}

// ---- GEMV launch ---------------------------------------------------------------------------
typedef void (*gemv_fn)(const GemvParams);

// The kernel of epilogue epi in one GEMV family for weights W: fam(std::integral_constant<int, EPI>(),
// type_tag<KV>()) names the family's instance.  KV is the context's store type for EPI_QKV, the one epilogue
// that writes the cache, and float otherwise.  EPI_XCHG (tensor parallel) has kernels only for fp32 weights
// (bf16 and q8 weights are single-GPU) and only in the families that declare it (XCHG); nullptr where there
// is no kernel.
template <typename W, bool XCHG, typename F>
gemv_fn pick_epi(const l2b_ctx *ctx, int epi, F fam) {
    auto f32 = type_tag<float>();
    switch (epi) {
    case EPI_STORE: return fam(std::integral_constant<int, EPI_STORE>(), f32);
    case EPI_ARGMAX: return fam(std::integral_constant<int, EPI_ARGMAX>(), f32);
    case EPI_QKV: return with_kv_store(ctx, [&fam](auto kv) { return fam(std::integral_constant<int, EPI_QKV>(), kv); });
    case EPI_SILU: return fam(std::integral_constant<int, EPI_SILU>(), f32);
    case EPI_XCHG:
        if constexpr (XCHG && std::is_same<W, float>::value) return fam(std::integral_constant<int, EPI_XCHG>(), f32);
        return nullptr;
    case EPI_RESID: return fam(std::integral_constant<int, EPI_RESID>(), f32);
    }
    return nullptr;
}
// the latency kernel's instance for tpr threads per row pair
template <int EPI, typename W, typename KV>
gemv_fn gemv_pick(int tpr) {
    switch (tpr) {
    case 8: return gemv_kernel<8, EPI, W, KV>;
    case 16: return gemv_kernel<16, EPI, W, KV>;
    case 32: return gemv_kernel<32, EPI, W, KV>;
    case 64: return gemv_kernel<64, EPI, W, KV>;
    case 128: return gemv_kernel<128, EPI, W, KV>;
    case 256: return gemv_kernel<256, EPI, W, KV>;
    }
    return nullptr;
}

constexpr int kMaxDynSmem = 200 * 1024;
constexpr size_t kDefaultDynSmem = 48 * 1024;       // a kernel's dynamic shared memory without an opt-in
constexpr int kMaxSmemOptin = 227 * 1024 - 2048;   // static __shared__ of the kernels stays under 2 KB

int gemv_tpr(int n) {
    const int n4 = n / 4;
    int tpr = 8;
    while (tpr < 256 && tpr * 2 <= n4 / 2) tpr *= 2;
    return tpr;
}

int prof_mark(l2b_ctx *ctx, const char *name, int layer, uint64_t bytes, cudaStream_t st) {
    if (!ctx->profiling) return L2B_OK;
    cudaEvent_t ev;
    L2B_CUDA(ctx, cudaEventCreate(&ev));
    L2B_CUDA(ctx, cudaEventRecord(ev, st));
    ctx->prof_ev.push_back(ev);
    l2b_kernel_time r{};
    snprintf(r.name, sizeof r.name, "%s", name);
    r.layer = layer;
    r.bytes = bytes;
    ctx->prof_rec.push_back(r);
    return L2B_OK;
}

// GEMV kernel families: the latency kernel (gemv_kernel, tpr threads per row pair), the register-fed
// 8-row kernel and the TMA ring
enum GemvKind { GK_LATENCY, GK_ROWS8, GK_TMA };

// The one place a GEMV kernel is chosen for the context's weight format and KV store; nullptr where the
// format has none.  The shape rules that pick `kind` are the same for every format (computed at 4 bytes
// per weight).
gemv_fn pick_gemv(const l2b_ctx *ctx, GemvKind kind, int epi, int tpr) {
    return with_w(ctx->wfmt, [&](auto w) -> gemv_fn {
        using W = typename decltype(w)::type;
        switch (kind) {
        case GK_LATENCY:
            return pick_epi<W, true>(ctx, epi, [tpr](auto e, auto kv) { return gemv_pick<decltype(e)::value, W, typename decltype(kv)::type>(tpr); });
        case GK_ROWS8:
            return pick_epi<W, true>(ctx, epi, [](auto e, auto kv) { return (gemv_fn)gemv8_kernel<decltype(e)::value, W, typename decltype(kv)::type>; });
        case GK_TMA:
            return pick_epi<W, true>(ctx, epi, [](auto e, auto kv) { return (gemv_fn)gemv_tma_kernel<decltype(e)::value, W, typename decltype(kv)::type>; });
        }
        return nullptr;
    });
}

cudaLaunchAttribute pdl_attr() {
    cudaLaunchAttribute at{};
    at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at.val.programmaticStreamSerializationAllowed = 1;
    return at;
}

unsigned long long *trace_slot(l2b_ctx *ctx) {
    if (!ctx->trace || ctx->profiling) return nullptr;
    return ctx->trace + (size_t)(ctx->last_launches % ctx->trace_launches) * TRACE_MAX_CTAS * TRACE_SLOTS;
}

// Ring slots of slot_bytes (at most max_slots) that fit next to xbytes of activation vectors under a
// dynamic shared-memory budget.  Compared before subtracting: (budget - xbytes) in unsigned
// arithmetic wraps once xbytes exceeds the budget.
int tma_ring_stages(size_t budget, size_t xbytes, size_t slot_bytes, int max_slots) {
    const int n = xbytes < budget ? (int)((budget - xbytes) / slot_bytes) : 0;
    return n < max_slots ? n : max_slots;
}
// the batched-prefill kernel's ring: stages of 8 rows (32 KB)
int pf_ring_stages(size_t budget, size_t xbytes) {
    return tma_ring_stages(budget, xbytes, (size_t)TMA_STAGE_FLOATS * 4, PF_MAX_STAGES);
}

int launch_gemv(l2b_ctx *ctx, int epi, const GemvParams &p, cudaStream_t st, const char *name = "gemv",
                int layer = -1) {
    {
        int prc = prof_mark(ctx, name, layer, (uint64_t)p.total_rows * w_ld(ctx, p.n) * w_elem(ctx), st);
        if (prc) return prc;
    }
    const size_t xbytes = (size_t)p.n * 4 * (1 + (p.gamma ? 1 : 0) + (p.parts ? 1 : 0));
    const size_t xonly = (size_t)p.n * 4;
    const size_t slot_bytes = with_w(ctx->wfmt, [](auto w) { return (size_t)DecodeRing<typename decltype(w)::type>::SLOT_BYTES; });
    // Decision from the shape.  Bandwidth-bound shapes take the TMA-ring kernel, latency-bound ones
    // the fine-grained kernel.  The ring kernel stages only x in shared memory; the rest of the
    // opt-in limit is its ring of 16 KB slots (13 next to a 16 KB x; DESIGN.md §4.1).
    bool big = ctx->gemv8_min_bytes >= 0 && p.n >= ctx->big_min_n &&
               (uint64_t)p.total_rows * p.n * 4ull >= (uint64_t)ctx->gemv8_min_bytes;
    int nstage = tma_ring_stages(kMaxSmemOptin, xonly, slot_bytes, TMA_MAX_STAGES);
    // Overrides: l2b_op_fused_matmul's kernel flavour, L2B_TMA_STAGES, L2B_GEMV_BIG=ldg (the
    // register-fed 8-row kernel for big shapes).
    if (ctx->force_kernel == 1) big = false;
    if (ctx->force_kernel >= 2) big = true;
    if (ctx->tma_stages > 0) nstage = ctx->tma_stages < TMA_MAX_STAGES ? ctx->tma_stages : TMA_MAX_STAGES;
    const bool fused_ok = !p.gamma || p.n <= TMA_MAXV * TMA_PRO_THREADS * 4;   // register slices of the rmsnorm gain
    bool tma = big && ctx->big_kernel_tma && nstage >= 2 && fused_ok && p.head_size <= 256 &&
               (size_t)nstage * slot_bytes + xonly <= (size_t)kMaxSmemOptin;
    if (ctx->force_kernel == 2) tma = false;
    // Hard invariants, whatever was decided above.
    if (p.parts && big) return fail(ctx, L2B_ERR_UNSUPPORTED, "partial-vector prologue is only in the latency kernel");
    if (ctx->force_kernel == 3 && !tma) return fail(ctx, L2B_ERR_UNSUPPORTED, "shape does not fit the TMA-ring kernel");
    const size_t smem = tma ? (size_t)nstage * slot_bytes + xonly : xbytes;
    if (smem > (size_t)kMaxSmemOptin) return fail(ctx, L2B_ERR_UNSUPPORTED, "activation vector too large for shared memory");
    if (tma && nstage < 2) return fail(ctx, L2B_ERR_UNSUPPORTED, "TMA ring of fewer than 2 stages");
    const int tpr = gemv_tpr(p.n);
    gemv_fn fn = pick_gemv(ctx, tma ? GK_TMA : big ? GK_ROWS8 : GK_LATENCY, epi, tpr);
    if (!fn) return fail(ctx, L2B_ERR_UNSUPPORTED, "no kernel for this epilogue in the context's weight format");
    if (!ctx->attr_done.count((const void *)fn)) {
        L2B_CUDA(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemOptin));
        ctx->attr_done.insert((const void *)fn);
    }
    const int threads = tma ? TMA_THREADS : NT;
    int occ = 0;
    L2B_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, threads, smem));
    if (occ < 1) occ = 1;
    if (tma) occ = 1;                        // the ring kernel is persistent: one CTA per SM walks that SM's rows
    int grid = ctx->num_sms * occ;
    if (big) {
        const int npairs = (p.total_rows + 1) / 2;
        if (grid > npairs) grid = npairs;
    } else {
        const int tile_rows = (NT / tpr) * GEMV_R;
        const int ntiles = (p.total_rows + tile_rows - 1) / tile_rows;
        if (grid > ntiles) grid = ntiles;
    }
    if (grid < 1) grid = 1;
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(grid);
    lc.blockDim = dim3(threads);
    lc.dynamicSmemBytes = smem;
    lc.stream = st;
    cudaLaunchAttribute at[1] = {pdl_attr()};
    lc.attrs = at;
    lc.numAttrs = ctx->use_pdl ? 1 : 0;
    GemvParams pp = p;
    pp.nstage = nstage;
    pp.nprefill = (ctx->tma_prefill > 0 && ctx->tma_prefill < nstage) ? ctx->tma_prefill : nstage;
    pp.spin_ns = ctx->spin_ns;
    pp.trace = trace_slot(ctx);
    ctx->last_grid = grid;
    L2B_CUDA(ctx, cudaLaunchKernelEx(&lc, fn, pp));
    ++ctx->last_launches;
    return L2B_OK;
}

typedef void (*attn_fn)(const AttnParams, const AttnBatch);
typedef void (*attn_wo_fn)(const AttnWoParams);

// The flash-decoding shape of head_size: lpr lanes share a row, each holding nf float4; a CTA covers ng rows.
// The flash kernel's dynamic shared memory follows from it, and attn_wo_kernel's adds the CTA's
// unnormalised output with its M and L, and the merged head output (page staging apart: attn_request).
struct AttnShape { int nf; size_t flash_smem, wo_smem; };
AttnShape attn_shape(int head_size) {
    const int hs4 = head_size / 4;
    const int lpr = (hs4 % 8 == 0) ? 8 : (hs4 % 4 == 0) ? 4 : (hs4 % 2 == 0) ? 2 : 1;
    const size_t ng = NWARP * (32 / lpr);
    const size_t flash = (ng * head_size + 3 * ng) * sizeof(float);
    return {hs4 / lpr, flash, flash + (2 * (size_t)head_size + 4) * sizeof(float)};
}
// f(std::integral_constant<int, NF>()) for the flash kernels' nf in {1..6, 8}; nullptr for any other nf
template <typename Fn, typename F>
Fn with_nf(int nf, F f) {
    switch (nf) {
    case 1: return f(std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>());
    case 3: return f(std::integral_constant<int, 3>());
    case 4: return f(std::integral_constant<int, 4>());
    case 5: return f(std::integral_constant<int, 5>());
    case 6: return f(std::integral_constant<int, 6>());
    case 8: return f(std::integral_constant<int, 8>());
    }
    return nullptr;
}

// flash-decoding form for KV when head_size has one (*smem: its request), else the 3-pass kernel
template <typename KV = float>
attn_fn pick_attention(int head_size, bool flash, size_t *smem) {
    const AttnShape sh = attn_shape(head_size);
    attn_fn f = nullptr;
    if (flash) f = with_nf<attn_fn>(sh.nf, [](auto nf) { return attention_flash_kernel<decltype(nf)::value, KV>; });
    if (!f) return attention_kernel<KV>;
    *smem = sh.flash_smem;
    return f;
}
// the instance for the context's cache (which kernel it is does not depend on the cache)
attn_fn pick_attention(const l2b_ctx *ctx, bool flash) {
    size_t unused = 0;
    return with_kv_read(ctx, [&](auto kv) { return pick_attention<typename decltype(kv)::type>(ctx->head_size, flash, &unused); });
}

// the attention + wo kernel for head_size, weights W and cache type KV; nullptr where head_size has no
// flash form
template <typename W = float, typename KV = float>
attn_wo_fn pick_attn_wo(int head_size) {
    return with_nf<attn_wo_fn>(attn_shape(head_size).nf, [](auto nf) { return attn_wo_kernel<decltype(nf)::value, W, KV>; });
}
// the instance for the context's weights and cache (whether one exists depends on neither)
attn_wo_fn pick_attn_wo(const l2b_ctx *ctx) {
    return with_w(ctx->wfmt, [ctx](auto w) {
        return with_kv_read(ctx, [ctx](auto kv) { return pick_attn_wo<typename decltype(w)::type, typename decltype(kv)::type>(ctx->head_size); });
    });
}

constexpr int kAttnClusterCtas = 8;   // CTAs per head cluster of attn_wo_kernel; 4 and 2 measured slower (DESIGN.md §4.6)

// The dynamic shared memory an attention kernel requests on ctx, page staging included: the 3-pass kernel
// (score buffer), the flash kernel (pick_attention: the 3-pass kernel's where the head size has no flash
// form) and attn_wo_kernel.  create_run_state checks and opts in these sizes and the launches request
// them, so the two cannot disagree.
enum AttnKind { ATTN_3PASS, ATTN_FLASH, ATTN_WO };
size_t attn_request(const l2b_ctx *ctx, AttnKind k) {
    if (k == ATTN_WO) return attn_shape(ctx->head_size).wo_smem + (ctx->paged ? ctx->attn_pg_bytes_wo : 0);
    size_t smem = ctx->attn_smem;
    pick_attention(ctx->head_size, k == ATTN_FLASH, &smem);
    return smem + (ctx->paged ? ctx->attn_pg_bytes : 0);
}

// attention + wo of one layer in one cluster launch (small models): partial vectors -> ctx->attn_parts
int launch_attn_wo(l2b_ctx *ctx, int layer, cudaStream_t st) {
    if (ctx->profiling) {
        const int hpos = ctx->n_appended > 0 ? ctx->n_appended - 1 : 0;
        int prc = prof_mark(ctx, "attn_wo", layer, 2ull * (uint64_t)(hpos + 1) * ctx->kv_loc * kv_elem(ctx) + (uint64_t)ctx->dim * w_ld(ctx, ctx->q_loc) * w_elem(ctx), st);
        if (prc) return prc;
    }
    AttnWoParams q{};
    AttnParams &a = q.a;
    a.ctl = ctx->ctl;
    a.q = ctx->q;
    a.kcache = kv_layer(ctx, ctx->kcache, layer);
    a.vcache = kv_layer(ctx, ctx->vcache, layer);
    a.head_size = ctx->head_size;
    a.kv_dim = ctx->kv_loc;
    a.kv_mul = ctx->kv_mul;
    a.trace = nullptr;
    a.kv_scale = kv_scale_at(ctx, layer);
    q.wo =wrow(ctx, ctx->wo, (uint64_t)layer * ctx->dim, ctx->q_loc);
    q.parts = ctx->attn_parts;
    q.dim = ctx->dim;
    q.q_dim = ctx->q_loc;
    attn_wo_fn fn = pick_attn_wo(ctx);
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(ctx->heads_loc, kAttnClusterCtas);
    lc.blockDim = dim3(NT);
    lc.dynamicSmemBytes = attn_request(ctx, ATTN_WO);
    lc.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = kAttnClusterCtas; at[0].val.clusterDim.z = 1;
    at[1] = pdl_attr();
    lc.attrs = at;
    lc.numAttrs = ctx->use_pdl ? 2 : 1;
    L2B_CUDA(ctx, cudaLaunchKernelEx(&lc, fn, q));
    ++ctx->last_launches;
    return L2B_OK;
}

// Attention of one layer for nb queries (gridDim.z).  Decode (zb == nullptr): one query at the control
// block's position on this context's caches.  Batched: query z at position zb->pos[z] on the caches
// zb->kcache[z] / vcache[z], q_stride floats apart in q and xb, with its own partial buffers and
// counters; it is not traced.
int launch_attention(l2b_ctx *ctx, int layer, cudaStream_t st, const float *q, float *xb, float *part_o,
                     float *part_ml, unsigned int *counters, const AttnBatch *zb = nullptr, int q_stride = 0,
                     int nb = 1) {
    if (ctx->profiling) {
        const int hpos = ctx->n_appended > 0 ? ctx->n_appended - 1 : 0;
        int prc = prof_mark(ctx, "attention", layer, 2ull * (uint64_t)(hpos + 1) * ctx->kv_loc * kv_elem(ctx), st);
        if (prc) return prc;
    }
    AttnParams a{};
    a.ctl = ctx->ctl;
    a.q = q;
    a.kcache = kv_layer(ctx, ctx->kcache, layer);
    a.vcache = kv_layer(ctx, ctx->vcache, layer);
    a.xb = xb;
    a.part_o = part_o;
    a.part_ml = part_ml;
    a.counters = counters;
    a.head_size = ctx->head_size;
    a.kv_dim = ctx->kv_loc;
    a.kv_mul = ctx->kv_mul;
    a.nsplit = ctx->nsplit;
    a.min_chunk = ctx->min_chunk;
    a.batched = zb ? 1 : 0;
    a.q_stride = q_stride;
    a.seq_len = ctx->cfg.seq_len;
    a.kv_scale = kv_scale_at(ctx, layer);
    a.trace = zb ? nullptr : trace_slot(ctx);
    const AttnBatch none{};
    attn_fn fn = pick_attention(ctx, ctx->attn_flash);
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(ctx->heads_loc, ctx->nsplit, nb);
    lc.blockDim = dim3(NT);
    lc.dynamicSmemBytes = attn_request(ctx, ctx->attn_flash ? ATTN_FLASH : ATTN_3PASS);
    lc.stream = st;
    cudaLaunchAttribute at[1] = {pdl_attr()};
    lc.attrs = at;
    lc.numAttrs = ctx->use_pdl ? 1 : 0;
    L2B_CUDA(ctx, cudaLaunchKernelEx(&lc, fn, a, zb ? *zb : none));
    ++ctx->last_launches;
    return L2B_OK;
}

// ---- tensor-parallel landing areas (offsets into an arena; same layout on every rank) --------
unsigned long long *ll_red_at(unsigned char *arena, const l2b_ctx *c, int slot, int src_rank) {
    return reinterpret_cast<unsigned long long *>(arena + c->off_red) + ((size_t)slot * c->world + src_rank) * c->dim;
}
unsigned long long *ll_logits_at(unsigned char *arena, const l2b_ctx *c) {
    return reinterpret_cast<unsigned long long *>(arena + c->off_logits);
}
unsigned long long *ll_amax_at(unsigned char *arena, const l2b_ctx *c, int src_rank) {
    return reinterpret_cast<unsigned long long *>(arena + c->off_amax) + 2 * (size_t)src_rank;
}


int launch_small(l2b_ctx *ctx, const void *fn, dim3 grid, dim3 block, void **args, cudaStream_t st, bool pdl) {
    cudaLaunchConfig_t lc{};
    lc.gridDim = grid;
    lc.blockDim = block;
    lc.stream = st;
    cudaLaunchAttribute at[1] = {pdl_attr()};
    lc.attrs = at;
    lc.numAttrs = (pdl && ctx->use_pdl) ? 1 : 0;
    L2B_CUDA(ctx, cudaLaunchKernelExC(&lc, fn, args));
    ++ctx->last_launches;
    return L2B_OK;
}

int launch_advance(l2b_ctx *ctx, cudaStream_t st, bool forced, bool exchange) {
    AdvanceParams a{};
    a.ctl = ctx->ctl;
    a.amax = ctx->amax;
    a.forced = forced ? ctx->gen_forced : nullptr;
    a.out_next = ctx->gen_out;
    a.n_done = ctx->gen_ndone;
    a.world = exchange ? ctx->world : 1;
    a.rank = ctx->rank;
    a.spin_ns = ctx->spin_ns;
    if (exchange) {
        for (int r = 0; r < ctx->world; ++r) a.ll_out[r] = ll_amax_at(ctx->peer_arena[r], ctx, ctx->rank);
        a.ll_in = ll_amax_at(ctx->arena, ctx, 0);
    }
    void *args[] = {&a};
    return launch_small(ctx, (const void *)advance_kernel, dim3(1), dim3(32), args, st, true);
}

// The four GEMVs of layer l, as the decode step and batched prefill share them: columns, rmsnorm gains,
// weights and row counts, and for qkv the caches, RoPE table and head size.  Inputs, outputs and
// whatever else is per launch are the caller's.
struct LayerGemvs {
    GemvParams qkv, wo, w13, w2;
};
LayerGemvs layer_gemvs(const l2b_ctx *ctx, int l) {
    const int dim = ctx->dim;
    LayerGemvs g{};
    // rmsnorm + q,k,v + RoPE + KV append (:305-358)
    GemvParams &p = g.qkv;
    p.ctl = ctx->ctl;
    p.n = dim;
    p.gamma = ctx->rms_att + (size_t)l * dim;
    p.w0 = wrow(ctx, ctx->wq, (uint64_t)l * ctx->q_loc, dim);
    p.w1 = wrow(ctx, ctx->wk, (uint64_t)l * ctx->kv_loc, dim);
    p.w2 = wrow(ctx, ctx->wv, (uint64_t)l * ctx->kv_loc, dim);
    p.rows0 = ctx->q_loc; p.rows1 = ctx->kv_loc; p.rows2 = ctx->kv_loc;
    p.total_rows = ctx->q_loc + 2 * ctx->kv_loc;
    p.kcache = kv_layer(ctx, ctx->kcache, l);
    p.vcache = kv_layer(ctx, ctx->vcache, l);
    p.rope_cos = ctx->rope_cos; p.rope_sin = ctx->rope_sin;
    p.head_size = ctx->head_size; p.kv_dim = ctx->kv_loc;
    p.kv_scale = kv_scale_at(ctx, l);
    // wo, whose result is added to the residual stream (:392-395)
    g.wo.ctl = ctx->ctl;
    g.wo.n = ctx->q_loc;
    g.wo.w0 = wrow(ctx, ctx->wo, (uint64_t)l * dim, ctx->q_loc);
    g.wo.total_rows = dim; g.wo.rows0 = dim;
    // rmsnorm + w1,w3 + SiLU*mul (:398-416)
    g.w13.ctl = ctx->ctl;
    g.w13.n = dim;
    g.w13.gamma = ctx->rms_ffn + (size_t)l * dim;
    g.w13.w0 = wrow(ctx, ctx->w1, (uint64_t)l * ctx->hid_loc, dim);
    g.w13.w1 = wrow(ctx, ctx->w3, (uint64_t)l * ctx->hid_loc, dim);
    g.w13.rows0 = ctx->hid_loc;
    g.w13.total_rows = 2 * ctx->hid_loc;
    // w2, added to the residual stream (:419-422)
    g.w2.ctl = ctx->ctl;
    g.w2.n = ctx->hid_loc;
    g.w2.w0 = wrow(ctx, ctx->w2, (uint64_t)l * dim, ctx->hid_loc);
    g.w2.total_rows = dim; g.w2.rows0 = dim;
    return g;
}

// One decode step on `st` (transformer(), src/main.zig:285-430).  All (token, pos) dependence is
// through ctx->ctl, so the sequence is capturable once and replayed.
int enqueue_step(l2b_ctx *ctx, cudaStream_t st, StepMode mode) {
    const l2b_config &c = ctx->cfg;
    const int dim = ctx->dim;
    const bool tp = ctx->world > 1;
    const bool p2p = tp && ctx->use_p2p;
    // my partial rows go to every rank; slice owners then fold all ranks' rows into x (tp_reduce_tail)
    auto produce_slot = [&](GemvParams &g, int slot, float *x) {
        g.ll_ndst = ctx->world;
        for (int r = 0; r < ctx->world; ++r) g.ll_out[r] = ll_red_at(ctx->peer_arena[r], ctx, slot, ctx->rank);
        g.ll_in = ll_red_at(ctx->arena, ctx, slot, 0);
        g.xres = x;
        g.xworld = ctx->world;
    };
    // wo / w2: row-parallel GEMV whose result is added to the residual stream (:392-395, :419-422)
    auto residual_gemv = [&](GemvParams &g, float *x, int slot, const char *name, int l) -> int {
        int rc;
        if (!tp) {
            g.out0 = x;
            rc = launch_gemv(ctx, EPI_RESID, g, st, name, l);
        } else if (p2p) {
            produce_slot(g, slot, x);
            rc = launch_gemv(ctx, EPI_XCHG, g, st, name, l);
        } else {
            g.out0 = ctx->delta;
            rc = launch_gemv(ctx, EPI_STORE, g, st, name, l);
            if (rc) return rc;
            L2B_NCCL(ctx, g_nccl.AllReduce(ctx->delta, ctx->delta, dim, ncclFloat, ncclSum, ctx->comm, st));
            resid_add_kernel<<<(dim + NT - 1) / NT, NT, 0, st>>>(x, ctx->delta, dim, ctx->ctl);
            L2B_CUDA(ctx, cudaGetLastError());
            ++ctx->last_launches;
        }
        return rc;
    };
    // small-model fusion (world == 1): attention+wo leaves its result as one partial vector per head
    // that the NEXT kernel's prologue sums into x; such a kernel reads x from one buffer and CTA 0
    // writes the new x to the other (ping-pong), everything else updates x in place
    float *Xc = ctx->X, *Xo = ctx->Xalt;
    const float *pend = nullptr;             // partial vectors still to be folded into x
    int npend = 0;

    auto fold_pending = [&](GemvParams &g) {
        g.x_in = Xc;
        if (pend) {
            g.parts = pend; g.nparts = npend; g.x_out = Xo;
            float *t = Xc; Xc = Xo; Xo = t;
            pend = nullptr; npend = 0;
        }
    };
    for (int l = 0; l < c.n_layers; ++l) {
        LayerGemvs g = layer_gemvs(ctx, l);
        // ---- rmsnorm + q,k,v + RoPE + KV append (:305-358)
        fold_pending(g.qkv);
        if (l == 0) {
            g.qkv.emb = ctx->emb;             // :295-296
            g.qkv.x_out = Xc;
            g.qkv.bump_epoch = 1;
        }
        g.qkv.out0 = ctx->q;
        int rc = launch_gemv(ctx, EPI_QKV, g.qkv, st, "qkv_rope", l);
        if (rc) return rc;

        if (ctx->fuse_attn) {
            // ---- attention + wo in one cluster launch (:361-392); the add of :395 happens in the next prologue
            rc = launch_attn_wo(ctx, l, st);
            if (rc) return rc;
            pend = ctx->attn_parts; npend = ctx->heads_loc;
        } else {
            // ---- attention (:361-389)
            rc = launch_attention(ctx, l, st, ctx->q, ctx->xb, ctx->part_o, ctx->part_ml, ctx->counters);
            if (rc) return rc;
            // ---- wo + residual (:392-395)
            g.wo.x_in = ctx->xb;
            rc = residual_gemv(g.wo, Xc, 2 * l, "wo", l);
            if (rc) return rc;
        }

        // ---- rmsnorm + w1,w3 + SiLU*mul (:398-416)
        fold_pending(g.w13);
        g.w13.out0 = ctx->hb;
        rc = launch_gemv(ctx, EPI_SILU, g.w13, st, "w13_silu", l);
        if (rc) return rc;

        // ---- w2 + residual (:419-422)
        g.w2.x_in = ctx->hb;
        rc = residual_gemv(g.w2, Xc, 2 * l + 1, "w2", l);
        if (rc) return rc;
    }
    if (mode == MODE_NOCLS) {   // prompt prefill: the logits of this position are never looked at (:996-1000)
        ctx->final_X = Xc;
        return L2B_OK;
    }
    // ---- final rmsnorm + classifier (:426-429)
    GemvParams k{};
    k.ctl = ctx->ctl;
    k.n = dim;
    fold_pending(k);
    ctx->final_X = Xc;
    k.gamma = ctx->rms_final;
    k.w0 = ctx->wcls;
    k.total_rows = ctx->vocab_loc; k.rows0 = ctx->vocab_loc;
    k.out0 = tp ? ctx->logits_loc : ctx->logits;
    k.amax = ctx->amax;
    k.row_base = ctx->rank * ctx->vocab_loc;
    const bool want_argmax = (mode == MODE_ARGMAX);
    int epi = want_argmax ? EPI_ARGMAX : EPI_STORE;
    const bool in_process = ctx->leader != nullptr;
    if (p2p && !want_argmax) {
        // logits slices travel as LL units: to every rank (one process per GPU: each rank's caller gets
        // the logits), or to rank 0 only (in-process group: one caller)
        epi = EPI_XCHG;
        if (in_process) {
            k.ll_ndst = 1;
            k.ll_out[0] = ll_logits_at(ctx->peer_arena[0], ctx);
        } else {
            k.ll_ndst = ctx->world;
            for (int r = 0; r < ctx->world; ++r) k.ll_out[r] = ll_logits_at(ctx->peer_arena[r], ctx);
        }
    }
    int rc = launch_gemv(ctx, epi, k, st, "classifier", -1);
    if (rc) return rc;
    if (tp) {
        if (p2p) {
            if (!want_argmax && (!in_process || ctx->rank == 0)) {
                float *lg = ctx->logits;
                const unsigned long long *in = ll_logits_at(ctx->arena, ctx);
                int V = c.vocab_size;
                const int *ctl = ctx->ctl;
                unsigned long long spin = ctx->spin_ns;
                void *args[] = {&lg, &in, &V, &ctl, &spin};
                int blocks = (V / 2 + NT - 1) / NT;
                if (blocks > ctx->num_sms) blocks = ctx->num_sms;
                rc = launch_small(ctx, (const void *)gather_logits_kernel, dim3(blocks), dim3(NT), args, st, true);
                if (rc) return rc;
            }
        } else if (want_argmax) {
            L2B_NCCL(ctx, g_nccl.AllReduce(ctx->amax, ctx->amax, 1, ncclUint64, ncclMax, ctx->comm, st));
        } else {
            L2B_NCCL(ctx, g_nccl.AllGather(ctx->logits_loc, ctx->logits, ctx->vocab_loc, ncclFloat, ctx->comm, st));
        }
    }
    return L2B_OK;
}

int launch_sample_prep(l2b_ctx *ctx, cudaStream_t st) {
    float *lg = ctx->logits;
    int V = ctx->cfg.vocab_size;
    const int *ctl = ctx->ctl;
    ProbIndex *cand = ctx->cand;
    int cap = kCandCap;
    int *n_cand = ctx->n_cand;
    void *args[] = {&lg, &V, &ctl, &cand, &cap, &n_cand};
    return launch_small(ctx, (const void *)sample_prep_kernel, dim3(1), dim3(SAMP_THREADS), args, st, true);
}

int launch_logprob(l2b_ctx *ctx, cudaStream_t st) {
    const float *lg = ctx->logits;
    int V = ctx->cfg.vocab_size;
    const int *ctl = ctx->ctl;
    const int *forced = ctx->gen_forced;
    const unsigned long long *amax = ctx->amax;
    float *lp = ctx->score_lp;
    int *greedy = ctx->score_greedy;
    void *args[] = {&lg, &V, &ctl, &forced, &amax, &lp, &greedy};
    return launch_small(ctx, (const void *)logprob_kernel, dim3(1), dim3(LOGPROB_THREADS), args, st, true);
}

// everything one call needs, as it is captured into (or eagerly enqueued instead of) graph `which`
int enqueue_call(l2b_ctx *ctx, cudaStream_t st, int which) {
    const bool sink = !ctx->leader || ctx->rank == 0;   // in-process group: only rank 0 returns data to the host
    // (token, pos) advance on the device
    const bool loop = (which == G_ARGMAX_LOOP || which == G_PREFILL_LOOP || which == G_SCORE_LOOP);
    if (!loop)
        L2B_CUDA(ctx, cudaMemcpyAsync(ctx->ctl, ctx->h_ctl, CTL_HOST_WORDS * sizeof(int), cudaMemcpyHostToDevice, st));
    const StepMode mode = (which == G_LOGITS) ? MODE_LOGITS : (which == G_SAMPLE) ? MODE_SAMPLE
                          : (which == G_PREFILL_LOOP) ? MODE_NOCLS : MODE_ARGMAX;
    int rc = enqueue_step(ctx, st, mode);
    if (rc) return rc;
    const size_t vbytes = (size_t)ctx->cfg.vocab_size * sizeof(float);
    switch (which) {
    case G_LOGITS:
        if (sink) L2B_CUDA(ctx, cudaMemcpyAsync(ctx->h_logits, ctx->logits, vbytes, cudaMemcpyDeviceToHost, st));
        break;
    case G_SAMPLE:
        if (sink) {
            rc = launch_sample_prep(ctx, st);
            if (rc) return rc;
            L2B_CUDA(ctx, cudaMemcpyAsync(ctx->h_logits, ctx->logits, vbytes, cudaMemcpyDeviceToHost, st));
            L2B_CUDA(ctx, cudaMemcpyAsync(ctx->h_cand, ctx->cand, (size_t)kCandCap * sizeof(ProbIndex), cudaMemcpyDeviceToHost, st));
            L2B_CUDA(ctx, cudaMemcpyAsync(ctx->h_ints + 2, ctx->n_cand, sizeof(int), cudaMemcpyDeviceToHost, st));
        }
        break;
    case G_ARGMAX_ONE:
        rc = launch_advance(ctx, st, false, ctx->world > 1 && ctx->use_p2p);
        if (rc) return rc;
        if (sink) L2B_CUDA(ctx, cudaMemcpyAsync(ctx->h_ints, ctx->gen_out, sizeof(int), cudaMemcpyDeviceToHost, st));
        break;
    case G_PREFILL_LOOP:   // every next token is forced: no argmax to exchange
        rc = launch_advance(ctx, st, true, false);
        if (rc) return rc;
        break;
    case G_SCORE_LOOP:     // single GPU only (l2b_score); every next token is forced
        rc = launch_logprob(ctx, st);
        if (rc) return rc;
        rc = launch_advance(ctx, st, true, false);
        if (rc) return rc;
        break;
    default:   // G_ARGMAX_LOOP
        rc = launch_advance(ctx, st, true, ctx->world > 1 && ctx->use_p2p);
        if (rc) return rc;
        break;
    }
    if (!loop && ctx->world > 1)   // the error word can only be raised by a tensor-parallel peer wait
        L2B_CUDA(ctx, cudaMemcpyAsync(ctx->h_ctl + CTL_WORDS, ctx->ctl, CTL_WORDS * sizeof(int), cudaMemcpyDeviceToHost, st));
    return L2B_OK;
}

int build_graphs(l2b_ctx *ctx) {
    for (int which = 0; which < G_COUNT; ++which) {
        if (which == G_SCORE_LOOP && ctx->world > 1) continue;   // l2b_score refuses tensor parallel
        cudaGraph_t g = nullptr;
        L2B_CUDA(ctx, cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed));
        ctx->last_launches = 0;
        int rc = enqueue_call(ctx, ctx->stream, which);
        cudaError_t e = cudaStreamEndCapture(ctx->stream, &g);
        if (rc) { if (g) cudaGraphDestroy(g); return rc; }
        L2B_CUDA(ctx, e);
        L2B_CUDA(ctx, cudaGraphInstantiate(&ctx->graphs[which], g, 0));
        L2B_CUDA(ctx, cudaGraphDestroy(g));
        if (which == G_LOGITS) ctx->launches_per_step = ctx->last_launches;
    }
    return L2B_OK;
}

int check_step_args(l2b_ctx *ctx, int token, int pos) {
    if (!ctx) return L2B_ERR_INVALID_ARG;
    if (token < 0 || token >= ctx->cfg.vocab_size) return fail(ctx, L2B_ERR_INVALID_ARG, "token out of range");
    if (pos < 0 || pos >= ctx->cfg.seq_len) return fail(ctx, L2B_ERR_INVALID_ARG, "pos out of range");
    if (pos > ctx->n_appended) return fail(ctx, L2B_ERR_STATE, "pos skips ahead of the KV cache");
    return L2B_OK;
}

#define L2B_TRY(expr)                                  \
    do {                                               \
        int rc__ = (expr);                             \
        if (rc__) {                                    \
            g_create_error = ctx->err;                 \
            return rc__;                               \
        }                                              \
    } while (0)

int cuda_try(l2b_ctx *ctx, cudaError_t e, const char *what) {
    if (e == cudaSuccess) return L2B_OK;
    ctx->err = std::string(what) + ": " + cudaGetErrorString(e);
    return e == cudaErrorMemoryAllocation ? L2B_ERR_OOM : L2B_ERR_CUDA;
}

// Load every kernel this library can launch onto the current device NOW.  With CUDA's default lazy
// module loading a kernel is loaded at its first launch, which can need the device to go idle —
// and a tensor-parallel kernel that is spinning on a peer (which the same host thread has not
// launched yet, in-process groups) would then never let it.
int preload_kernels(l2b_ctx *ctx) {
    cudaFuncAttributes fa;
    const int tprs[] = {8, 16, 32, 64, 128, 256};
    for (int epi = 0; epi < EPI_COUNT; ++epi) {
        if (!pick_gemv(ctx, GK_TMA, epi, 0)) continue;   // EPI_XCHG: no kernel in a bf16 or q8 family
        for (int tpr : tprs) L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)pick_gemv(ctx, GK_LATENCY, epi, tpr)));
        L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)pick_gemv(ctx, GK_ROWS8, epi, 0)));
        L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)pick_gemv(ctx, GK_TMA, epi, 0)));
    }
    L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)pick_attention(ctx, true)));
    if (attn_wo_fn aw = pick_attn_wo(ctx)) L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)aw));
    const void *fork = with_kv_elem(ctx->kvfmt, [](auto e) { return (const void *)kv_fork_kernel<typename decltype(e)::type>; });
    const void *others[] = {(const void *)pick_attention(ctx, false), (const void *)advance_kernel,
                            (const void *)batch_advance_kernel, (const void *)gather_logits_kernel,
                            (const void *)resid_add_kernel, (const void *)sample_prep_kernel,
                            (const void *)sample_prep_batch_kernel, (const void *)logprob_kernel,
                            (const void *)logprob_batch_kernel, (const void *)logprob_topk_batch_kernel,
                            (const void *)synth_fill_kernel,
                            (const void *)synth_fill_bf16_kernel, (const void *)synth_fill_q8_kernel,
                            fork, (const void *)verify_accept_kernel};
    for (const void *f : others) L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, f));
    // The kernels that run next to a TMA-ring GEMV in a decode step (the ring GEMVs, attention, the
    // token advance) all ask for the largest shared-memory carveout, so consecutive kernels never
    // need a different L1 / shared split on an SM.  (A successor was not seen to enter an SM early
    // for it, DESIGN.md §4.1; what dropping the attribute costs or gains is not measured.)
    const void *decode[] = {(const void *)pick_attention(ctx, true), (const void *)pick_attention(ctx, false),
                            (const void *)advance_kernel};
    for (const void *f : decode)
        L2B_CUDA(ctx, cudaFuncSetAttribute(f, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    for (int epi = 0; epi < EPI_COUNT; ++epi)
        if (gemv_fn f = pick_gemv(ctx, GK_TMA, epi, 0))
            L2B_CUDA(ctx, cudaFuncSetAttribute((const void *)f, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    return L2B_OK;
}

// ---- creation, stage 1: weights + run state of one rank (no peer is touched) ------------------
// device, derived sizes, stream and events of one rank
int init_rank(l2b_ctx *ctx, const l2b_config *cfg, int rank, int world, int device) {
    cudaDeviceProp prop{};
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { ctx->err = "cudaGetDeviceProperties failed"; g_create_error = ctx->err; return L2B_ERR_CUDA; }
    if (prop.major != 9 || prop.minor != 0) { ctx->err = "device is not compute capability 9.0 (built for sm_90a only)"; g_create_error = ctx->err; return L2B_ERR_NO_DEVICE; }
    ctx->cfg = *cfg;
    ctx->rank = rank; ctx->world = world; ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    ctx->dim = cfg->dim; ctx->hidden = cfg->hidden_dim;
    ctx->head_size = cfg->dim / cfg->n_heads;
    ctx->kv_mul = cfg->n_heads / cfg->n_kv_heads;
    ctx->q_dim = cfg->dim;
    ctx->kv_dim = ctx->head_size * cfg->n_kv_heads;
    ctx->q_loc = ctx->q_dim / world; ctx->kv_loc = ctx->kv_dim / world;
    ctx->hid_loc = cfg->hidden_dim / world;
    ctx->heads_loc = cfg->n_heads / world;
    ctx->vocab_loc = cfg->vocab_size / world;

    L2B_TRY(cuda_try(ctx, cudaSetDevice(device), "cudaSetDevice"));
    L2B_TRY(cuda_try(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking), "cudaStreamCreate"));
    L2B_TRY(cuda_try(ctx, cudaEventCreate(&ctx->ev0), "cudaEventCreate"));
    L2B_TRY(cuda_try(ctx, cudaEventCreate(&ctx->ev1), "cudaEventCreate"));
    L2B_TRY(preload_kernels(ctx));
    return L2B_OK;
}

int create_run_state(l2b_ctx *ctx);

int create_rank(l2b_ctx *ctx, const l2b_config *cfg, const Source &src, const float *rope_cos,
                const float *rope_sin, int rank, int world, int device) {
    L2B_TRY(init_rank(ctx, cfg, rank, world, device));
    ctx->weights = new SharedWeights();
    const uint64_t dim = cfg->dim, hid = cfg->hidden_dim, L = cfg->n_layers, V = cfg->vocab_size, S = cfg->seq_len;
    const uint64_t hs = ctx->head_size, kvd = ctx->kv_dim;
    const double sd = sqrt(288.0 / (double)dim), sh = sqrt(768.0 / (double)hid);
    const float BIG = 3.0e38f;
    // payload offsets in checkpoint order (src/main.zig:85-112)
    uint64_t off = 0;
    const uint64_t o_emb = off;  off += V * dim;
    const uint64_t o_ratt = off; off += L * dim;
    const uint64_t o_wq = off;   off += L * dim * dim;
    const uint64_t o_wk = off;   off += L * kvd * dim;
    const uint64_t o_wv = off;   off += L * kvd * dim;
    const uint64_t o_wo = off;   off += L * dim * dim;
    const uint64_t o_rffn = off; off += L * dim;
    const uint64_t o_w1 = off;   off += L * hid * dim;
    const uint64_t o_w2 = off;   off += L * dim * hid;
    const uint64_t o_w3 = off;   off += L * hid * dim;
    const uint64_t o_rfin = off; off += dim;
    off += 2 * (S * hs / 2);     // freq_cis_real/imag: not used by transformer() (:67-69, :298-300)
    const uint64_t o_wcls = off;

    const auto t_load0 = std::chrono::steady_clock::now();
    L2B_TRY(materialize(ctx, &ctx->emb, src, o_emb, 1, 1, V, dim, SH_NONE, {0.0, 0.04, -BIG, BIG}, true));
    L2B_TRY(materialize(ctx, &ctx->rms_att, src, o_ratt, 2, 1, L, dim, SH_NONE, {1.35, 0.35, 0.25f, 2.4f}));
    L2B_TRY(materialize(ctx, &ctx->wq, src, o_wq, 3, L, dim, dim, SH_ROWS, {0.0, 0.04 * sd, -BIG, BIG}, true));
    L2B_TRY(materialize(ctx, &ctx->wk, src, o_wk, 4, L, kvd, dim, SH_ROWS, {0.0, 0.04 * sd, -BIG, BIG}, true));
    L2B_TRY(materialize(ctx, &ctx->wv, src, o_wv, 5, L, kvd, dim, SH_ROWS, {0.0, 0.02 * sd, -BIG, BIG}, true));
    L2B_TRY(materialize(ctx, &ctx->wo, src, o_wo, 6, L, dim, dim, SH_COLS, {0.0, 0.02 * sd, -BIG, BIG}, true));
    L2B_TRY(materialize(ctx, &ctx->rms_ffn, src, o_rffn, 7, 1, L, dim, SH_NONE, {1.35, 0.35, 0.25f, 2.4f}));
    L2B_TRY(materialize(ctx, &ctx->w1, src, o_w1, 8, L, hid, dim, SH_ROWS, {0.0, 0.026 * sd, -BIG, BIG}, true));
    L2B_TRY(materialize(ctx, &ctx->w2, src, o_w2, 9, L, dim, hid, SH_COLS, {0.0, 0.026 * sh, -BIG, BIG}, true));
    L2B_TRY(materialize(ctx, &ctx->w3, src, o_w3, 10, L, hid, dim, SH_ROWS, {0.0, 0.026 * sd, -BIG, BIG}, true));
    L2B_TRY(materialize(ctx, &ctx->rms_final, src, o_rfin, 11, 1, 1, dim, SH_NONE, {7.1, 0.6, 3.0f, 10.0f}));
    if (cfg->shared_weights) {
        ctx->wcls = const_cast<void *>(wrow(ctx, ctx->emb, (uint64_t)rank * ctx->vocab_loc, dim));   // :112
    } else {
        L2B_TRY(materialize(ctx, &ctx->wcls, src, o_wcls, 14, 1, V, dim, SH_ROWS, {0.0, 0.04, -BIG, BIG}, true));
    }
    if (ctx->d_rounded) {
        unsigned long long n = 0;
        L2B_TRY(cuda_try(ctx, cudaMemcpyAsync(&n, ctx->d_rounded, sizeof n, cudaMemcpyDeviceToHost, ctx->stream), "rounding count"));
        L2B_TRY(cuda_try(ctx, cudaStreamSynchronize(ctx->stream), "weight upload"));
        ctx->n_rounded = n;
    }
    L2B_TRY(cuda_try(ctx, cudaStreamSynchronize(ctx->stream), "weight upload"));
    ctx->load_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_load0).count();
    for (int i = 0; i < 2; ++i) {          // the staging buffers are only needed during the upload
        if (ctx->stage[i]) { cudaFreeHost(ctx->stage[i]); ctx->stage[i] = nullptr; }
        if (ctx->stage_ev[i]) { cudaEventDestroy(ctx->stage_ev[i]); ctx->stage_ev[i] = nullptr; }
    }

    // ---- RoPE table (:338-342); the host's own libm values when the caller passes them
    L2B_TRY(dev_alloc(ctx, &ctx->rope_cos, S * hs / 2, &ctx->weights->owned));
    L2B_TRY(dev_alloc(ctx, &ctx->rope_sin, S * hs / 2, &ctx->weights->owned));
    {
        std::vector<float> hc(S * hs / 2), hsn(S * hs / 2);
        if (rope_cos && rope_sin) {
            memcpy(hc.data(), rope_cos, hc.size() * sizeof(float));
            memcpy(hsn.data(), rope_sin, hsn.size() * sizeof(float));
        } else {
            for (uint64_t p = 0; p < S; ++p)
                for (uint64_t j = 0; j < hs / 2; ++j) {
                    const float head_dim = (float)(2 * j);                                   // i % head_size
                    const float freq = 1.0f / powf(10000.0f, head_dim / (float)hs);          // :339
                    const float val = (float)p * freq;                                       // :340
                    hc[p * (hs / 2) + j] = cosf(val);                                        // :341
                    hsn[p * (hs / 2) + j] = sinf(val);                                       // :342
                }
        }
        L2B_TRY(cuda_try(ctx, cudaMemcpy(ctx->rope_cos, hc.data(), hc.size() * sizeof(float), cudaMemcpyHostToDevice), "rope upload"));
        L2B_TRY(cuda_try(ctx, cudaMemcpy(ctx->rope_sin, hsn.data(), hsn.size() * sizeof(float), cudaMemcpyHostToDevice), "rope upload"));
    }
    if (kv_scaled(ctx->kvfmt)) {                 // the e4m3 scales, 1 until l2b_kv_scales
        SharedWeights *w = ctx->weights;
        w->kv_scale_h.assign(2 * L, 1.0f);
        L2B_TRY(dev_alloc(ctx, &w->kv_scale, 2 * L, &w->owned));
        L2B_TRY(cuda_try(ctx, cudaMemcpy(w->kv_scale, w->kv_scale_h.data(), 2 * L * sizeof(float), cudaMemcpyHostToDevice), "KV scale upload"));
    }
    return create_run_state(ctx);
}

// run state, attention launch shape, pinned host buffers, tensor-parallel landing area and switches
// of one rank whose weights are in place

// ---- paged KV (L2B_KV_PAGED): the model's page pool, each session's page table, and the reservation
// every writing call makes before it launches -----------------------------------------------------------
size_t kv_page_bytes(const l2b_ctx *ctx) { return 2ull * ctx->cfg.n_layers * KV_PAGE_ROWS * ctx->kv_loc * kv_elem(ctx); }
KvPool *kv_pool(const l2b_ctx *ctx) { return ctx->paged && ctx->weights ? ctx->weights->pool : nullptr; }

// host table entries of page index j for every layer: `page`, or the null page when nullptr
void kv_tab_set(l2b_ctx *ctx, int j, void *page) {
    unsigned char *base = static_cast<unsigned char *>(page ? page : kv_pool(ctx)->null_page);
    const size_t layer_bytes = 2ull * KV_PAGE_ROWS * ctx->kv_loc * kv_elem(ctx);
    for (int l = 0; l < ctx->cfg.n_layers; ++l) ctx->h_tab[(size_t)l * ctx->n_pages + j] = base + (size_t)l * layer_bytes;
    ctx->tab_dirty = true;
}
// The table goes up whole (n_layers * ceil(seq_len / P) addresses) and is synchronised: a batched call runs
// on its first session's stream, and the next kernel that reads this table may be on any of them.
int kv_tab_upload(l2b_ctx *ctx) {
    if (!ctx->tab_dirty) return L2B_OK;
    L2B_CUDA(ctx, cudaMemcpyAsync(ctx->kv_tab, ctx->h_tab, (size_t)ctx->cfg.n_layers * ctx->n_pages * sizeof(void *),
                                  cudaMemcpyHostToDevice, ctx->stream));
    L2B_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->tab_dirty = false;
    return L2B_OK;
}

// a session's page table (every entry on the null page) and, for the model's first context, the pool
int kv_paged_init(l2b_ctx *ctx) {
    SharedWeights *w = ctx->weights;
    if (!w->pool) {
        w->pool = new KvPool();
        w->pool->page_bytes = kv_page_bytes(ctx);
        L2B_CUDA(ctx, cudaMalloc(&w->pool->null_page, w->pool->page_bytes));
        L2B_CUDA(ctx, cudaMemset(w->pool->null_page, 0, w->pool->page_bytes));
    }
    ctx->n_pages = (ctx->cfg.seq_len + KV_PAGE_ROWS - 1) / KV_PAGE_ROWS;
    ctx->pages.assign(ctx->n_pages, nullptr);
    const size_t n = (size_t)ctx->cfg.n_layers * ctx->n_pages;
    int rc = dev_alloc(ctx, &ctx->kv_tab, n);
    if (rc) return rc;
    L2B_CUDA(ctx, cudaHostAlloc((void **)&ctx->h_tab, n * sizeof(void *), cudaHostAllocDefault));
    for (int j = 0; j < ctx->n_pages; ++j) kv_tab_set(ctx, j, nullptr);
    ctx->kcache = ctx->vcache = ctx->kv_tab;
    return kv_tab_upload(ctx);
}

int kv_page_get(l2b_ctx *ctx, KvPool *pool, void **out) {
    if (pool->limit && pool->refs.size() >= pool->limit) return fail(ctx, L2B_ERR_OOM, "the model's KV pages are all in use (l2b_kv_pool_limit)");
    void *pg = nullptr;
    if (!pool->free_pages.empty()) {
        pg = pool->free_pages.back();
        pool->free_pages.pop_back();
    } else {
        if (cudaMalloc(&pg, pool->page_bytes) != cudaSuccess) { cudaGetLastError(); return fail(ctx, L2B_ERR_OOM, "cudaMalloc of a KV page failed"); }
        pool->all.push_back(pg);
    }
    pool->refs[pg] = 1;
    *out = pg;
    return L2B_OK;
}
void kv_page_put(KvPool *pool, void *pg) {
    auto it = pool->refs.find(pg);
    if (--it->second == 0) {
        pool->refs.erase(it);
        pool->free_pages.push_back(pg);
    }
}
// session ctx gives up page j
void kv_drop(l2b_ctx *ctx, int j) {
    if (!ctx->pages[j]) return;
    kv_page_put(kv_pool(ctx), ctx->pages[j]);
    ctx->pages[j] = nullptr;
    kv_tab_set(ctx, j, nullptr);
}
// kv_fork_kernel on ctx's stream: in every layer l, the segments of seg elements at k + l * stride and
// v + l * stride into the same offsets from every destination pair dst[d] = (K base, V base), KV_FORK_MAXD
// destinations per launch.  One 4-element unit per thread: on llama2-7B (fp32) this grid beat one resident
// wave of grid-striding CTAs (8 per SM) by 5-12 % at every n_pos and destination count measured, and
// cudaMemcpy at one destination (DESIGN.md §4.5g).
int kv_fork_launch(l2b_ctx *ctx, const void *k, const void *v, long long seg, long long stride,
                   const std::vector<std::pair<void *, void *>> &dst) {
    return with_kv_elem(ctx->kvfmt, [&](auto e) -> int {
        using E = typename decltype(e)::type;
        KvForkParams<E> p{};
        p.k = static_cast<const E *>(k);
        p.v = static_cast<const E *>(v);
        p.seg = seg;
        p.stride = stride;
        p.L = ctx->cfg.n_layers;
        const int gy = std::min(2 * p.L, 65535);
        const int gx = (int)std::min(((seg >> 2) + NT - 1) / NT, (long long)INT32_MAX);
        for (size_t g = 0; g < dst.size(); g += KV_FORK_MAXD) {
            p.nd = (int)std::min(dst.size() - g, (size_t)KV_FORK_MAXD);
            for (int d = 0; d < p.nd; ++d) {
                p.dk[d] = static_cast<E *>(dst[g + d].first);
                p.dv[d] = static_cast<E *>(dst[g + d].second);
            }
            void *args[] = {&p};
            const int rc = launch_small(ctx, (const void *)kv_fork_kernel<E>, dim3(gx, gy), dim3(NT), args, ctx->stream, false);
            if (rc) return rc;
        }
        return L2B_OK;
    });
}
// Rows [0, rows) of every layer, K and V, of page src into the nd pages dst: one page as the "cache" (layers
// 2P rows apart, V rows P rows after K rows).
int kv_page_copy(l2b_ctx *ctx, const void *src, void *const *dst, int nd, int rows) {
    const long long half = (long long)KV_PAGE_ROWS * ctx->kv_loc;   // elements
    const size_t half_bytes = (size_t)half * kv_elem(ctx);
    std::vector<std::pair<void *, void *>> d;
    for (int i = 0; i < nd; ++i) d.emplace_back(dst[i], static_cast<unsigned char *>(dst[i]) + half_bytes);
    return kv_fork_launch(ctx, src, static_cast<const unsigned char *>(src) + half_bytes, (long long)rows * ctx->kv_loc, 2 * half, d);
}

// rows [lo, hi) that a call may write into session s's cache (a paged session; one call lists no other)
struct KvRange { l2b_ctx *s; int lo, hi; };

// The reservation every writing entry point makes after its argument checks and before it launches: for
// each session, the pages of its range that it does not hold are allocated, and those it shares with
// another session (reference count above 1) are replaced by private copies (copy-on-write).  Then every
// listed session's changed table goes up.  When a page cannot be had (the pool limit, or cudaMalloc) every
// page this reservation took is given back and L2B_ERR_OOM returned: no session has changed.
int kv_reserve(l2b_ctx *err_ctx, const std::vector<KvRange> &r) {
    if (r.empty() || !r[0].s->paged) return L2B_OK;
    L2B_CUDA(err_ctx, cudaSetDevice(r[0].s->device));
    struct Step { l2b_ctx *s; int j; void *old; };
    std::vector<Step> done;
    int rc = L2B_OK;
    for (const KvRange &x : r) {
        KvPool *pool = kv_pool(x.s);   // a target and its draft are two models
        const int hi = std::min(x.hi, x.s->cfg.seq_len);
        for (int j = x.lo / KV_PAGE_ROWS; rc == L2B_OK && x.lo < hi && j <= (hi - 1) / KV_PAGE_ROWS; ++j) {
            void *old = x.s->pages[j];
            if (old && pool->refs[old] == 1) continue;
            void *pg = nullptr;
            rc = kv_page_get(err_ctx, pool, &pg);
            if (rc) break;
            if (old) --pool->refs[old];      // still held by another session: never 0 here
            x.s->pages[j] = pg;
            done.push_back(Step{x.s, j, old});
        }
        if (rc) break;
    }
    if (rc) {
        for (size_t i = done.size(); i-- > 0;) {
            const Step &d = done[i];
            kv_page_put(kv_pool(d.s), d.s->pages[d.j]);
            if (d.old) ++kv_pool(d.s)->refs[d.old];
            d.s->pages[d.j] = d.old;
        }
        return rc;
    }
    for (const Step &d : done) {
        if (d.old) {
            rc = kv_page_copy(d.s, d.old, &d.s->pages[d.j], 1, KV_PAGE_ROWS);
            if (rc) { err_ctx->err = d.s->err; return rc; }
        }
        kv_tab_set(d.s, d.j, d.s->pages[d.j]);
    }
    for (const KvRange &x : r) {
        rc = kv_tab_upload(x.s);   // synchronises the copies above too
        if (rc) { err_ctx->err = x.s->err; return rc; }
    }
    return L2B_OK;
}
// after a call: the pages wholly at or past the appended count go back to the pool
void kv_release(l2b_ctx *ctx) {
    if (!ctx->paged) return;
    for (int j = (ctx->n_appended + KV_PAGE_ROWS - 1) / KV_PAGE_ROWS; j < ctx->n_pages; ++j) kv_drop(ctx, j);
}
// A writing call's pages: reserve() before the first launch; every session it listed releases its pages
// past its appended count when the call returns, refused or not.
struct KvCall {
    std::vector<l2b_ctx *> s;
    KvCall() = default;
    KvCall(const KvCall &) = delete;
    ~KvCall() { for (l2b_ctx *c : s) kv_release(c); }
    int reserve(l2b_ctx *err_ctx, const std::vector<KvRange> &r) {
        for (const KvRange &x : r) s.push_back(x.s);
        return kv_reserve(err_ctx, r);
    }
};

int create_run_state(l2b_ctx *ctx) {
    const l2b_config *cfg = &ctx->cfg;
    const int rank = ctx->rank, world = ctx->world;
    const uint64_t dim = cfg->dim, L = cfg->n_layers, V = cfg->vocab_size, S = cfg->seq_len;
    const uint64_t hs = ctx->head_size;
    L2B_TRY(dev_alloc(ctx, &ctx->X, dim));
    L2B_TRY(dev_alloc(ctx, &ctx->Xalt, dim));
    {
        // small-model fusion: attention + wo as one cluster kernel (8 CTAs per head; 4 or 2 are slower
        // on H100) is +1.0 % on stories15M on H100 and +0.5 % on stories110M, too little there to change
        // its summation order, so it is on for dim <= 512 only (L2B_FUSE=0|1 overrides;
        // results/h100_policy_ab.txt)
        const char *ef = getenv("L2B_FUSE");
        const int want = ef ? atoi(ef) : (dim <= 512 ? 1 : 0);
        ctx->fuse_attn = (want & 1) && world == 1 && dim < 1024 && pick_attn_wo((int)hs) != nullptr;
        if (ctx->fuse_attn) L2B_TRY(dev_alloc(ctx, &ctx->attn_parts, (size_t)cfg->n_heads * dim));
    }
    L2B_TRY(dev_alloc(ctx, &ctx->delta, dim));
    L2B_TRY(dev_alloc(ctx, &ctx->q, (size_t)ctx->q_loc));
    L2B_TRY(dev_alloc(ctx, &ctx->xb, (size_t)ctx->q_loc));
    L2B_TRY(dev_alloc(ctx, &ctx->hb, (size_t)ctx->hid_loc));
    L2B_TRY(dev_alloc(ctx, &ctx->logits, V));
    if (world > 1) L2B_TRY(dev_alloc(ctx, &ctx->logits_loc, (size_t)ctx->vocab_loc));
    const size_t kv_bytes = ctx->paged ? 0 : L * S * ctx->kv_loc * kv_elem(ctx);
    if (ctx->paged) {
        L2B_TRY(kv_paged_init(ctx));
    } else {
        unsigned char *kc = nullptr, *vc = nullptr;
        L2B_TRY(dev_alloc(ctx, &kc, kv_bytes));
        L2B_TRY(dev_alloc(ctx, &vc, kv_bytes));
        ctx->kcache = kc; ctx->vcache = vc;
    }
    L2B_TRY(dev_alloc(ctx, &ctx->ctl, (size_t)CTL_WORDS));
    L2B_TRY(dev_alloc(ctx, &ctx->amax, (size_t)1));
    L2B_TRY(dev_alloc(ctx, &ctx->gen_forced, S));
    L2B_TRY(dev_alloc(ctx, &ctx->gen_out, S));
    L2B_TRY(dev_alloc(ctx, &ctx->gen_ndone, (size_t)1));
    L2B_TRY(dev_alloc(ctx, &ctx->cand, (size_t)kCandCap));
    L2B_TRY(dev_alloc(ctx, &ctx->n_cand, (size_t)1));
    L2B_TRY(dev_alloc(ctx, &ctx->score_lp, S));
    L2B_TRY(dev_alloc(ctx, &ctx->score_greedy, S));
    L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->ctl, 0, CTL_WORDS * sizeof(int), ctx->stream), "memset"));
    L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->X, 0, dim * sizeof(float), ctx->stream), "memset"));
    L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->amax, 0, sizeof(unsigned long long), ctx->stream), "memset"));
    L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->gen_forced, 0xff, S * sizeof(int), ctx->stream), "memset"));
    if (!ctx->paged) {
        L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->kcache, 0, kv_bytes, ctx->stream), "memset"));
        L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->vcache, 0, kv_bytes, ctx->stream), "memset"));
    }

    // ---- attention launch shape: enough (head, split) CTAs to cover the SMs, chunks >= min_chunk positions
    {
        const char *envc = getenv("L2B_ATTN_MIN_CHUNK");
        if (envc && atoi(envc) >= 8) ctx->min_chunk = atoi(envc);
        int ns = (2 * ctx->num_sms + ctx->heads_loc - 1) / ctx->heads_loc;
        const int max_by_len = (int)((S + ctx->min_chunk - 1) / ctx->min_chunk);
        if (ns > max_by_len) ns = max_by_len;
        if (ns > 32) ns = 32;
        if (ns < 1) ns = 1;
        ctx->nsplit = ns;
        int cap = (int)((S + ns - 1) / ns);
        if (cap < ctx->min_chunk) cap = ctx->min_chunk;
        const int G = NT / (int)(hs / 4);
        ctx->attn_smem = (int)(((uint64_t)G * hs + cap) * sizeof(float));
        // paged: each split's page addresses follow the kernels' shared memory (a split of `cap` rows
        // spans at most cap / P + 2 pages; attn_wo_kernel's splits are ceil(S / 8) rows)
        ctx->attn_pg_bytes = (int)(((size_t)cap / KV_PAGE_ROWS + 2) * sizeof(void *) + sizeof(float));
        ctx->attn_pg_bytes_wo = (int)(((S + kAttnClusterCtas - 1) / kAttnClusterCtas / KV_PAGE_ROWS + 2) * sizeof(void *));
        // every attention kernel this context can launch (the 3-pass one also under L2B_ATTN=3pass) must
        // get its request; the flash and attn_wo requests grow with seq_len only through page staging
        const size_t req_3pass = attn_request(ctx, ATTN_3PASS), req_flash = attn_request(ctx, ATTN_FLASH);
        const size_t req_wo = ctx->fuse_attn ? attn_request(ctx, ATTN_WO) : 0;
        if (std::max({req_3pass, req_flash, req_wo}) > (size_t)kMaxDynSmem) {
            ctx->err = "seq_len too large for the attention kernel's shared memory";
            g_create_error = ctx->err;
            return L2B_ERR_UNSUPPORTED;
        }
        L2B_TRY(cuda_try(ctx, cudaFuncSetAttribute(pick_attention(ctx, false), cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem), "cudaFuncSetAttribute"));
        // past the 48 KiB a kernel gets without opting in (long paged contexts only); kMaxDynSmem, as for
        // the 3-pass kernel, so another context's smaller request never lowers it
        if (req_flash > kDefaultDynSmem)
            L2B_TRY(cuda_try(ctx, cudaFuncSetAttribute(pick_attention(ctx, true), cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem), "cudaFuncSetAttribute"));
        if (req_wo > kDefaultDynSmem)
            L2B_TRY(cuda_try(ctx, cudaFuncSetAttribute(pick_attn_wo(ctx), cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem), "cudaFuncSetAttribute"));
        L2B_TRY(dev_alloc(ctx, &ctx->part_o, (size_t)ctx->heads_loc * ns * hs));
        L2B_TRY(dev_alloc(ctx, &ctx->part_ml, (size_t)ctx->heads_loc * ns * 2));
        L2B_TRY(dev_alloc(ctx, &ctx->counters, (size_t)ctx->heads_loc));
        L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->counters, 0, ctx->heads_loc * sizeof(unsigned int), ctx->stream), "memset"));
    }

    // ---- pinned host buffers
    L2B_TRY(cuda_try(ctx, cudaHostAlloc((void **)&ctx->h_logits, V * sizeof(float), cudaHostAllocDefault), "cudaHostAlloc"));
    L2B_TRY(cuda_try(ctx, cudaHostAlloc((void **)&ctx->h_ctl, 2 * CTL_WORDS * sizeof(int), cudaHostAllocDefault), "cudaHostAlloc"));
    L2B_TRY(cuda_try(ctx, cudaHostAlloc((void **)&ctx->h_ints, 16 * sizeof(int), cudaHostAllocDefault), "cudaHostAlloc"));
    L2B_TRY(cuda_try(ctx, cudaHostAlloc((void **)&ctx->h_gen, S * sizeof(int), cudaHostAllocDefault), "cudaHostAlloc"));
    L2B_TRY(cuda_try(ctx, cudaHostAlloc((void **)&ctx->h_cand, (size_t)kCandCap * sizeof(ProbIndex), cudaHostAllocDefault), "cudaHostAlloc"));
    memset(ctx->h_ctl, 0, 2 * CTL_WORDS * sizeof(int));

    // ---- tensor-parallel landing areas: one zeroed arena
    if (world > 1) {
        const size_t slots = 2 * (size_t)L;
        size_t o = 0;
        ctx->off_red = o;    o += slots * world * dim * sizeof(unsigned long long);
        ctx->off_logits = o; o += (size_t)V * sizeof(unsigned long long);
        ctx->off_amax = o;   o += (size_t)world * 2 * sizeof(unsigned long long);
        ctx->arena_bytes = (o + 255) & ~(size_t)255;
        L2B_TRY(dev_alloc(ctx, &ctx->arena, ctx->arena_bytes));
        L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->arena, 0, ctx->arena_bytes, ctx->stream), "memset"));
        ctx->peer_arena[rank] = ctx->arena;
    }

    {
        const char *env = getenv("L2B_NO_GRAPH");
        ctx->use_graphs = !(env && env[0] == '1');
        const char *env2 = getenv("L2B_NO_PDL");
        ctx->use_pdl = !(env2 && env2[0] == '1');
        const char *envts = getenv("L2B_TIME_STEPS");
        ctx->time_steps = envts && envts[0] == '1';
        const char *env3 = getenv("L2B_GEMV8_MIN_BYTES");
        if (env3) ctx->gemv8_min_bytes = atoll(env3);
        const char *env4 = getenv("L2B_GEMV_BIG");
        if (env4 && strcmp(env4, "ldg") == 0) ctx->big_kernel_tma = false;
        const char *env5 = getenv("L2B_TMA_STAGES");
        if (env5) ctx->tma_stages = atoi(env5);
        const char *enva = getenv("L2B_ATTN");
        if (enva && strcmp(enva, "3pass") == 0) ctx->attn_flash = false;
        const char *envpf = getenv("L2B_TMA_PREFILL");
        if (envpf) ctx->tma_prefill = atoi(envpf);
        const char *envs = getenv("L2B_SPIN_TIMEOUT_MS");
        if (envs && atoll(envs) > 0) ctx->spin_ns = (unsigned long long)atoll(envs) * 1000000ull;
        const char *envt = getenv("L2B_TRACE");
        if (envt && envt[0] == '1') {
            ctx->trace_launches = 5 * cfg->n_layers + 4;
            L2B_TRY(dev_alloc(ctx, &ctx->trace, (size_t)ctx->trace_launches * TRACE_MAX_CTAS * TRACE_SLOTS));
            L2B_TRY(cuda_try(ctx, cudaMemset(ctx->trace, 0, (size_t)ctx->trace_launches * TRACE_MAX_CTAS * TRACE_SLOTS * 8), "memset"));
        }
        const char *envn = getenv("L2B_BIG_MIN_N");
        if (envn && atoi(envn) >= 4) ctx->big_min_n = atoi(envn);
    }
    L2B_TRY(cuda_try(ctx, cudaStreamSynchronize(ctx->stream), "cudaStreamSynchronize"));
    return L2B_OK;
}

// ---- creation, stage 2: one eager call of each flavour on every local rank.  It sets function
// attributes outside capture and surfaces launch errors before a graph hides them (it scribbles
// on KV row 0, rewritten by step 0).  Tensor-parallel ranks exchange data during these steps, so
// all local ranks are enqueued before any is synchronised.
int warm_up(const std::vector<l2b_ctx *> &ranks) {
    for (int which = 0; which < G_COUNT; ++which) {
        if (which == G_SCORE_LOOP && ranks[0]->world > 1) continue;   // as build_graphs
        for (l2b_ctx *ctx : ranks) {
            L2B_TRY(cuda_try(ctx, cudaSetDevice(ctx->device), "cudaSetDevice"));
            memset(ctx->h_ctl, 0, CTL_WORDS * sizeof(int));
            ctx->h_ctl[CTL_TEMP] = 0x3f800000;   // 1.0f
            ctx->h_ctl[CTL_TOPP] = 0x3f666666;   // 0.9f
            if (which == G_ARGMAX_LOOP || which == G_PREFILL_LOOP || which == G_SCORE_LOOP)
                L2B_TRY(cuda_try(ctx, cudaMemcpyAsync(ctx->ctl, ctx->h_ctl, CTL_HOST_WORDS * sizeof(int), cudaMemcpyHostToDevice, ctx->stream), "ctl upload"));
            L2B_TRY(enqueue_call(ctx, ctx->stream, which));
        }
        for (l2b_ctx *ctx : ranks) {
            L2B_TRY(cuda_try(ctx, cudaSetDevice(ctx->device), "cudaSetDevice"));
            L2B_TRY(cuda_try(ctx, cudaStreamSynchronize(ctx->stream), "warm-up step"));
            L2B_TRY(cuda_try(ctx, cudaGetLastError(), "warm-up step"));
            if (ctx->h_ctl[CTL_WORDS + CTL_ERR] && which != G_ARGMAX_LOOP && which != G_PREFILL_LOOP &&
                which != G_SCORE_LOOP) {
                ctx->err = "tensor-parallel warm-up step timed out waiting for a peer";
                g_create_error = ctx->err;
                return L2B_ERR_COMM;
            }
        }
    }
    for (l2b_ctx *ctx : ranks) {
        L2B_TRY(cuda_try(ctx, cudaSetDevice(ctx->device), "cudaSetDevice"));
        if (ctx->use_graphs) L2B_TRY(build_graphs(ctx));
    }
    return L2B_OK;
}

// ---- one process per GPU: communicator + CUDA IPC exchange of the arena handles ---------------
int connect_ipc(l2b_ctx *ctx, const l2b_shard *shard) {
    const int world = ctx->world, rank = ctx->rank;
    std::string e;
    if (!nccl_load(&e)) { ctx->err = e; g_create_error = e; return L2B_ERR_COMM; }
    ncclUniqueId id;
    memcpy(&id, shard->comm_id, sizeof id);
    ncclResult_t r = g_nccl.CommInitRank(&ctx->comm, world, id, rank);
    if (r != ncclSuccess) {
        ctx->err = std::string("ncclCommInitRank: ") + g_nccl.GetErrorString(r);
        g_create_error = ctx->err;
        return L2B_ERR_COMM;
    }
    const char *mode = getenv("L2B_TP");
    const bool want = !(mode && strcmp(mode, "nccl") == 0);
    int ok = want ? 1 : 0;
    cudaIpcMemHandle_t hx{};
    if (ok && cudaIpcGetMemHandle(&hx, ctx->arena) != cudaSuccess) {
        cudaGetLastError();
        ok = 0;
    }
    // every rank learns every rank's handle (and whether it could make one) through NCCL
    struct Msg { cudaIpcMemHandle_t hx; int ok; int pad[3]; };
    static_assert(sizeof(Msg) % 16 == 0, "Msg must be 16-byte sized");
    Msg mine{hx, ok, {0, 0, 0}};
    Msg *d_all = nullptr;
    L2B_TRY(dev_alloc(ctx, &d_all, (size_t)world));
    L2B_TRY(cuda_try(ctx, cudaMemcpyAsync(d_all + rank, &mine, sizeof(Msg), cudaMemcpyHostToDevice, ctx->stream), "msg upload"));
    if (g_nccl.AllGather(d_all + rank, d_all, sizeof(Msg), ncclChar, ctx->comm, ctx->stream) != ncclSuccess) {
        ctx->err = "ncclAllGather(ipc handles) failed"; g_create_error = ctx->err; return L2B_ERR_COMM;
    }
    std::vector<Msg> all(world);
    L2B_TRY(cuda_try(ctx, cudaMemcpyAsync(all.data(), d_all, sizeof(Msg) * world, cudaMemcpyDeviceToHost, ctx->stream), "msg download"));
    L2B_TRY(cuda_try(ctx, cudaStreamSynchronize(ctx->stream), "ipc exchange"));
    for (int q = 0; q < world; ++q) ok = ok && all[q].ok;
    if (ok) {
        for (int q = 0; q < world && ok; ++q) {
            if (q == rank) continue;
            void *px = nullptr;
            if (cudaIpcOpenMemHandle(&px, all[q].hx, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                cudaGetLastError();
                ok = 0;
                break;
            }
            ctx->ipc_opened.push_back(px);
            ctx->peer_arena[q] = (unsigned char *)px;
        }
    }
    // all ranks must take the same path: agree through a max-reduce of the failure bit
    int *d_bad = nullptr;
    L2B_TRY(dev_alloc(ctx, &d_bad, (size_t)1));
    int bad = ok ? 0 : 1;
    L2B_TRY(cuda_try(ctx, cudaMemcpyAsync(d_bad, &bad, sizeof(int), cudaMemcpyHostToDevice, ctx->stream), "flag upload"));
    if (g_nccl.AllReduce(d_bad, d_bad, 1, ncclInt, ncclMax, ctx->comm, ctx->stream) != ncclSuccess) {
        ctx->err = "ncclAllReduce(ipc agreement) failed"; g_create_error = ctx->err; return L2B_ERR_COMM;
    }
    L2B_TRY(cuda_try(ctx, cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream), "flag download"));
    L2B_TRY(cuda_try(ctx, cudaStreamSynchronize(ctx->stream), "ipc agreement"));
    ctx->use_p2p = (bad == 0);
    return L2B_OK;
}

void destroy_rank(l2b_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    // graphs first: NCCL keeps a communicator alive (ncclCommDestroy spins) while captured
    // graphs still reference it
    for (int i = 0; i < G_COUNT; ++i)
        if (ctx->graphs[i]) cudaGraphExecDestroy(ctx->graphs[i]);
    cudaDeviceSynchronize();
    if (ctx->comm && g_nccl.ok) g_nccl.CommDestroy(ctx->comm);
    for (void *p : ctx->ipc_opened) cudaIpcCloseMemHandle(p);
    for (void *p : ctx->owned) cudaFree(p);
    if (kv_pool(ctx))
        for (int j = 0; j < ctx->n_pages; ++j)
            if (ctx->pages[j]) kv_page_put(kv_pool(ctx), ctx->pages[j]);
    if (ctx->weights && --ctx->weights->refs == 0) {   // the last context or session of the model
        for (void *p : ctx->weights->owned) cudaFree(p);
        if (KvPool *pool = ctx->weights->pool) {
            for (void *p : pool->all) cudaFree(p);
            if (pool->null_page) cudaFree(pool->null_page);
            delete pool;
        }
        delete ctx->weights;
    }
    for (int i = 0; i < 2; ++i) {
        if (ctx->stage[i]) cudaFreeHost(ctx->stage[i]);
        if (ctx->stage_ev[i]) cudaEventDestroy(ctx->stage_ev[i]);
    }
    if (ctx->h_logits) cudaFreeHost(ctx->h_logits);
    if (ctx->h_ctl) cudaFreeHost(ctx->h_ctl);
    if (ctx->h_ints) cudaFreeHost(ctx->h_ints);
    if (ctx->h_gen) cudaFreeHost(ctx->h_gen);
    if (ctx->h_cand) cudaFreeHost(ctx->h_cand);
    if (ctx->h_call) cudaFreeHost(ctx->h_call);
    if (ctx->h_tab) cudaFreeHost(ctx->h_tab);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

void destroy_all(l2b_ctx *ctx) {
    if (!ctx) return;
    std::vector<l2b_ctx *> ranks = locals(ctx);
    // every rank must be idle before any rank's memory (a peer's landing area) goes away
    for (l2b_ctx *c : ranks) { cudaSetDevice(c->device); if (c->stream) cudaStreamSynchronize(c->stream); }
    for (size_t i = ranks.size(); i-- > 0;) destroy_rank(ranks[i]);
}

// warm_up's step at position 0 wrote through a page table that holds no page: into the null page
int kv_null_clear(l2b_ctx *ctx) {
    if (KvPool *pool = kv_pool(ctx)) L2B_CUDA(ctx, cudaMemset(pool->null_page, 0, pool->page_bytes));
    return L2B_OK;
}

int common_create(l2b_ctx **out, const l2b_config *cfg, const Source &src, uint64_t n_floats,
                  const float *rope_cos, const float *rope_sin, const l2b_shard *shard, int n_gpus,
                  int wfmt = L2B_WEIGHTS_F32, int kvfmt = 0, bool paged = false) {
    if (!out || !cfg) { g_create_error = "NULL argument"; return L2B_ERR_INVALID_ARG; }
    *out = nullptr;
    const bool in_process = n_gpus > 1;
    const int world = shard ? shard->world_size : n_gpus;
    std::string why;
    int rc = validate_config(cfg, world, &why);
    if (rc) { g_create_error = why; return rc; }
    if (shard && (shard->rank < 0 || shard->rank >= world)) { g_create_error = "rank out of range"; return L2B_ERR_INVALID_ARG; }
    if (src.host && n_floats < checkpoint_floats(cfg)) {
        g_create_error = "host_weights shorter than the checkpoint layout requires";
        return L2B_ERR_INVALID_ARG;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        g_create_error = "no CUDA device";
        return L2B_ERR_NO_DEVICE;
    }
    if (in_process && ndev < n_gpus) { g_create_error = "fewer CUDA devices than n_gpus"; return L2B_ERR_NO_DEVICE; }
    const int device0 = shard ? shard->device : 0;
    if (device0 < 0 || device0 >= ndev) { g_create_error = "device ordinal out of range"; return L2B_ERR_INVALID_ARG; }

    std::vector<l2b_ctx *> ranks;
    auto bail = [&](int code) {
        for (size_t i = ranks.size(); i-- > 0;) destroy_rank(ranks[i]);
        return code;
    };
    const int nlocal = in_process ? n_gpus : 1;
    for (int i = 0; i < nlocal; ++i) {
        l2b_ctx *ctx = new l2b_ctx();
        ranks.push_back(ctx);
        ctx->wfmt = wfmt;
        ctx->kvfmt = kvfmt;
        ctx->paged = paged;
        const int rank = in_process ? i : (shard ? shard->rank : 0);
        const int device = in_process ? i : device0;
        rc = create_rank(ctx, cfg, src, rope_cos, rope_sin, rank, world, device);
        if (rc) return bail(rc);
    }
    if (in_process) {
        // one process drives all GPUs: peers are plain UVA pointers once peer access is on
        for (l2b_ctx *a : ranks) {
            cudaSetDevice(a->device);
            for (l2b_ctx *b : ranks) {
                if (a == b) continue;
                int can = 0;
                cudaDeviceCanAccessPeer(&can, a->device, b->device);
                if (!can) { g_create_error = "GPUs are not peer-accessible (NVLink/NVSwitch required for n_gpus > 1)"; return bail(L2B_ERR_COMM); }
                cudaError_t e = cudaDeviceEnablePeerAccess(b->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { g_create_error = std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e); return bail(L2B_ERR_COMM); }
                cudaGetLastError();
                a->peer_arena[b->rank] = b->arena;
            }
            a->use_p2p = true;
            a->leader = ranks[0];
        }
    } else if (world > 1) {
        rc = connect_ipc(ranks[0], shard);
        if (rc) return bail(rc);
    }
    rc = warm_up(ranks);
    if (rc) return bail(rc);
    rc = kv_null_clear(ranks[0]);
    if (rc) return bail(rc);
    if (in_process) ranks[0]->members = ranks;
    *out = ranks[0];
    return L2B_OK;
}

// a context on the weights of `model` (single GPU): its own run state, caches, stream and graphs
int create_session(l2b_ctx *ctx, const l2b_ctx *model) {
    ctx->wfmt = model->wfmt;
    ctx->kvfmt = model->kvfmt;
    ctx->paged = model->paged;
    ctx->n_rounded = model->n_rounded;
    L2B_TRY(init_rank(ctx, &model->cfg, 0, 1, model->device));
    ctx->weights = model->weights;
    ++ctx->weights->refs;
    ctx->emb = model->emb; ctx->rms_att = model->rms_att; ctx->rms_ffn = model->rms_ffn; ctx->rms_final = model->rms_final;
    ctx->wq = model->wq; ctx->wk = model->wk; ctx->wv = model->wv; ctx->wo = model->wo;
    ctx->w1 = model->w1; ctx->w2 = model->w2; ctx->w3 = model->w3; ctx->wcls = model->wcls;
    ctx->rope_cos = model->rope_cos; ctx->rope_sin = model->rope_sin;
    L2B_TRY(create_run_state(ctx));
    L2B_TRY(warm_up(std::vector<l2b_ctx *>{ctx}));
    return kv_null_clear(ctx);
}
#undef L2B_TRY

// ---- running a call on every local rank -------------------------------------------------------
void fill_ctl(l2b_ctx *ctx, int token, int pos, int stop_on_bos, float temperature, float top_p) {
    int *h = ctx->h_ctl;
    h[CTL_TOKEN] = token; h[CTL_POS] = pos; h[CTL_DONE] = 0; h[CTL_STEP] = 0;
    h[CTL_STOP_ON_BOS] = stop_on_bos;
    memcpy(&h[CTL_TEMP], &temperature, sizeof(float));
    memcpy(&h[CTL_TOPP], &top_p, sizeof(float));
}

// one synchronise of each rank's stream (ranks[0] is the lead, which keeps the error); with one rank
// the current device is already its own
int finish_call(l2b_ctx *const *ranks, size_t n) {
    l2b_ctx *lead = ranks[0];
    int rc = L2B_OK;
    for (size_t i = 0; i < n; ++i) {
        l2b_ctx *c = ranks[i];
        if (n > 1) cudaSetDevice(c->device);
        cudaError_t e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess && rc == L2B_OK) {
            lead->err = std::string("step failed: ") + cudaGetErrorString(e);
            rc = L2B_ERR_CUDA;
        }
        if (c->h_ctl[CTL_WORDS + CTL_ERR] && rc == L2B_OK) {
            lead->err = "tensor-parallel exchange timed out: a peer rank died or fell out of lockstep";
            rc = L2B_ERR_COMM;
        }
    }
    return rc;
}

// run one step; which: G_LOGITS / G_ARGMAX_ONE / G_SAMPLE
int run_step(l2b_ctx *lead, int token, int pos, int which, float temperature, float top_p) {
    // One step costs a small model ~90 us on the device, so every host call here is on the clock of
    // the end-to-end loop: no per-step events unless asked for (L2B_TIME_STEPS=1), no allocation.
    l2b_ctx *single[1] = {lead};
    l2b_ctx *const *ranks = lead->members.empty() ? single : lead->members.data();
    const size_t nranks = lead->members.empty() ? 1 : lead->members.size();
    KvCall kv;
    if (int rc = kv.reserve(lead, {{lead, pos, pos + 1}})) return rc;
    for (size_t i = 0; i < nranks; ++i) {
        l2b_ctx *ctx = ranks[i];
        if (nranks > 1 || i == 0) L2B_CUDA(lead, cudaSetDevice(ctx->device));
        fill_ctl(ctx, token, pos, 0, temperature, top_p);
        ctx->last_launches = 0;
        if (ctx == lead && lead->time_steps) L2B_CUDA(lead, cudaEventRecord(ctx->ev0, ctx->stream));
        if (ctx->use_graphs) {
            L2B_CUDA(lead, cudaGraphLaunch(ctx->graphs[which], ctx->stream));
            ctx->last_launches = ctx->launches_per_step + (which == G_LOGITS ? 0 : 1);
        } else {
            int rc = enqueue_call(ctx, ctx->stream, which);
            if (rc) { lead->err = ctx->err; return rc; }
        }
        if (ctx == lead && lead->time_steps) L2B_CUDA(lead, cudaEventRecord(ctx->ev1, ctx->stream));
    }
    int rc = finish_call(ranks, nranks);
    if (rc) return rc;
    if (lead->time_steps) {
        if (nranks > 1) L2B_CUDA(lead, cudaSetDevice(lead->device));
        L2B_CUDA(lead, cudaEventElapsedTime(&lead->last_ms, lead->ev0, lead->ev1));
    }
    if (pos + 1 > lead->n_appended) lead->n_appended = pos + 1;
    return L2B_OK;
}

// The output of a sampling step, from the pinned buffers it was copied to (V probabilities probs, the
// candidates h_cand and their count): the probabilities to host_probs (if not NULL and not probs itself),
// and with the candidate filter the candidates and their count to cand / *n_cand, or minus their number
// when more passed than fit (the host then filters the probabilities itself).  Without the filter *n_cand = 0.
void copy_sample_out(int V, const float *probs, const ProbIndex *h_cand, int count, bool filter, float *host_probs,
                     l2b_prob_index *cand, int cand_cap, int32_t *n_cand) {
    if (host_probs && host_probs != probs) memcpy(host_probs, probs, (size_t)V * sizeof(float));
    if (n_cand) *n_cand = 0;
    if (filter) {
        if (count > kCandCap || count > cand_cap) { *n_cand = -count; return; }   // too many: filter host_probs on the host
        static_assert(sizeof(l2b_prob_index) == sizeof(ProbIndex), "candidate layout");
        memcpy(cand, h_cand, (size_t)count * sizeof(ProbIndex));
        *n_cand = count;
    }
}
// the output of ctx's last single sampling step (G_SAMPLE), from its own pinned buffers
void copy_step_sample_out(l2b_ctx *ctx, bool filter, float *host_probs, l2b_prob_index *cand, int cand_cap, int32_t *n_cand) {
    copy_sample_out(ctx->cfg.vocab_size, ctx->h_logits, ctx->h_cand, ctx->h_ints[2], filter, host_probs, cand, cand_cap, n_cand);
}

}  // namespace

// ---------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------
extern "C" {

int32_t l2b_abi_version(void) { return L2B_ABI_VERSION; }

const char *l2b_status_string(int32_t s) {
    switch (s) {
    case L2B_OK: return "ok";
    case L2B_ERR_INVALID_ARG: return "invalid argument";
    case L2B_ERR_UNSUPPORTED: return "unsupported shape";
    case L2B_ERR_CUDA: return "CUDA error";
    case L2B_ERR_NO_DEVICE: return "no usable sm_90 device";
    case L2B_ERR_OOM: return "out of memory";
    case L2B_ERR_COMM: return "communication error";
    case L2B_ERR_STATE: return "call order violated";
    default: return "unknown status";
    }
}

const char *l2b_last_error(const l2b_ctx *ctx) {
    if (!ctx) return g_create_error.c_str();
    return ctx->err.empty() ? kNoError : ctx->err.c_str();
}

uint64_t l2b_checkpoint_floats(const l2b_config *cfg) { return cfg ? checkpoint_floats(cfg) : 0; }

int32_t l2b_create(l2b_ctx **out, const l2b_config *cfg, const float *host_weights, uint64_t n_floats,
                   const float *rope_cos, const float *rope_sin, int32_t n_gpus) {
    if (!host_weights) { g_create_error = "host_weights is NULL"; return L2B_ERR_INVALID_ARG; }
    if (n_gpus != 1 && n_gpus != 2 && n_gpus != 4 && n_gpus != 8) {
        g_create_error = "n_gpus must be 1, 2, 4 or 8";
        return L2B_ERR_UNSUPPORTED;
    }
    Source s; s.host = host_weights;
    return common_create(out, cfg, s, n_floats, rope_cos, rope_sin, nullptr, n_gpus);
}

int32_t l2b_create_sharded(l2b_ctx **out, const l2b_config *cfg, const float *host_weights,
                           uint64_t n_floats, const float *rope_cos, const float *rope_sin,
                           const l2b_shard *shard) {
    if (!host_weights || !shard) { g_create_error = "NULL argument"; return L2B_ERR_INVALID_ARG; }
    Source s; s.host = host_weights;
    return common_create(out, cfg, s, n_floats, rope_cos, rope_sin, shard, 1);
}

int32_t l2b_create_synthetic(l2b_ctx **out, const l2b_config *cfg, uint64_t seed, const l2b_shard *shard) {
    Source s; s.host = nullptr; s.seed = seed;
    return common_create(out, cfg, s, 0, nullptr, nullptr, shard, 1);
}

int32_t l2b_create_synthetic_group(l2b_ctx **out, const l2b_config *cfg, uint64_t seed, int32_t n_gpus) {
    if (n_gpus != 1 && n_gpus != 2 && n_gpus != 4 && n_gpus != 8) {
        g_create_error = "n_gpus must be 1, 2, 4 or 8";
        return L2B_ERR_UNSUPPORTED;
    }
    Source s; s.host = nullptr; s.seed = seed;
    return common_create(out, cfg, s, 0, nullptr, nullptr, nullptr, n_gpus);
}

// weight_format of l2b_create_format: a weight format, with at most one of L2B_KV_BF16, L2B_KV_ROUND_BF16,
// L2B_KV_E4M3 and L2B_KV_ROUND_E4M3 and optionally L2B_KV_PAGED or'd in; split into the weight format, the
// KV element format and the layout.  Any other value => L2B_ERR_INVALID_ARG.
bool split_format(int32_t weight_format, int *wfmt, int *kvfmt, bool *paged) {
    const int elem = L2B_KV_BF16 | L2B_KV_ROUND_BF16 | L2B_KV_E4M3 | L2B_KV_ROUND_E4M3;
    *kvfmt = weight_format & elem;
    *paged = (weight_format & L2B_KV_PAGED) != 0;
    *wfmt = weight_format & ~(elem | L2B_KV_PAGED);
    if ((*wfmt != L2B_WEIGHTS_F32 && *wfmt != L2B_WEIGHTS_BF16 && *wfmt != L2B_WEIGHTS_Q8) || (*kvfmt & (*kvfmt - 1)) != 0) {
        g_create_error = "unknown weight format";
        return false;
    }
    return true;
}

int32_t l2b_create_format(l2b_ctx **out, const l2b_config *cfg, const float *host_weights, uint64_t n_floats,
                          const float *rope_cos, const float *rope_sin, int32_t n_gpus, int32_t weight_format) {
    int wfmt, kvfmt;
    bool paged;
    if (!split_format(weight_format, &wfmt, &kvfmt, &paged)) return L2B_ERR_INVALID_ARG;
    if (weight_format == L2B_WEIGHTS_F32) return l2b_create(out, cfg, host_weights, n_floats, rope_cos, rope_sin, n_gpus);
    if (!host_weights) { g_create_error = "host_weights is NULL"; return L2B_ERR_INVALID_ARG; }
    if (n_gpus != 1) { g_create_error = "bf16 and q8 weights and bf16, e4m3 or paged KV caches are single-GPU (n_gpus must be 1)"; return L2B_ERR_UNSUPPORTED; }
    Source s; s.host = host_weights;
    return common_create(out, cfg, s, n_floats, rope_cos, rope_sin, nullptr, 1, wfmt, kvfmt, paged);
}

int32_t l2b_create_synthetic_format(l2b_ctx **out, const l2b_config *cfg, uint64_t seed, int32_t weight_format) {
    int wfmt, kvfmt;
    bool paged;
    if (!split_format(weight_format, &wfmt, &kvfmt, &paged)) return L2B_ERR_INVALID_ARG;
    Source s; s.host = nullptr; s.seed = seed;
    return common_create(out, cfg, s, 0, nullptr, nullptr, nullptr, 1, wfmt, kvfmt, paged);
}

int32_t l2b_kv_info(const l2b_ctx *ctx, int32_t *kv_format, uint64_t *cache_bytes) {
    if (!ctx) return L2B_ERR_INVALID_ARG;
    if (kv_format) *kv_format = ctx->kvfmt;
    if (cache_bytes && ctx->paged) {
        uint64_t held = 0;
        for (void *pg : ctx->pages) held += pg != nullptr;
        *cache_bytes = held * kv_page_bytes(ctx);
    } else if (cache_bytes) {
        *cache_bytes = 2ull * ctx->cfg.n_layers * ctx->cfg.seq_len * ctx->kv_loc * kv_elem(ctx);
    }
    return L2B_OK;
}

int32_t l2b_kv_pool_info(const l2b_ctx *ctx, int32_t *page_rows, uint64_t *page_bytes, uint64_t *pages_in_use,
                         uint64_t *pages_allocated) {
    if (!ctx || !page_rows || !page_bytes || !pages_in_use || !pages_allocated) return L2B_ERR_INVALID_ARG;
    const KvPool *pool = kv_pool(ctx);
    *page_rows = pool ? KV_PAGE_ROWS : 0;
    *page_bytes = pool ? pool->page_bytes : 0;
    *pages_in_use = pool ? pool->refs.size() : 0;
    *pages_allocated = pool ? pool->all.size() : 0;
    return L2B_OK;
}

int32_t l2b_kv_pool_limit(l2b_ctx *ctx, uint64_t max_pages) {
    if (!ctx) return L2B_ERR_INVALID_ARG;
    KvPool *pool = kv_pool(ctx);
    if (!pool) return fail(ctx, L2B_ERR_UNSUPPORTED, "the model's KV cache is not paged");
    if (max_pages && max_pages < pool->refs.size()) return fail(ctx, L2B_ERR_INVALID_ARG, "max_pages is below the pages in use");
    pool->limit = max_pages;
    return L2B_OK;
}

int32_t l2b_weight_info(const l2b_ctx *ctx, int32_t *weight_format, uint64_t *n_rounded) {
    if (!ctx) return L2B_ERR_INVALID_ARG;
    if (weight_format) *weight_format = ctx->wfmt;
    if (n_rounded) *n_rounded = ctx->n_rounded;
    return L2B_OK;
}

int32_t l2b_kv_scales(l2b_ctx *ctx, const float *scales, int32_t n) {
    if (!ctx) return L2B_ERR_INVALID_ARG;
    if (!scales) return fail(ctx, L2B_ERR_INVALID_ARG, "scales is NULL");
    if (n != 2 * ctx->cfg.n_layers) return fail(ctx, L2B_ERR_INVALID_ARG, "n must be 2 * n_layers");
    for (int i = 0; i < n; ++i)
        if (!std::isnormal(scales[i]) || !(scales[i] > 0.0f)) return fail(ctx, L2B_ERR_INVALID_ARG, "a KV scale is not a finite positive normal float");
    if (!kv_scaled(ctx->kvfmt)) return fail(ctx, L2B_ERR_UNSUPPORTED, "the model's KV cache is not e4m3");
    SharedWeights *w = ctx->weights;
    if (w->refs > 1) return fail(ctx, L2B_ERR_STATE, "the model has a live session");
    if (ctx->n_appended > 0) return fail(ctx, L2B_ERR_STATE, "the model has positions appended");
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    L2B_CUDA(ctx, cudaMemcpy(w->kv_scale, scales, (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
    w->kv_scale_h.assign(scales, scales + n);
    return L2B_OK;
}

void l2b_round_e4m3_host(float *data, uint64_t n, float scale) {
    if (!data) return;
    for (uint64_t i = 0; i < n; ++i) data[i] = e4m3_widen(e4m3_round_bits(data[i], scale), scale);
}

void l2b_round_bf16_host(float *data, uint64_t n) {
    if (!data) return;
    for (uint64_t i = 0; i < n; ++i) {
        uint32_t u;
        memcpy(&u, data + i, 4);
        u = (uint32_t)bf16_round_bits(u) << 16;
        memcpy(data + i, &u, 4);
    }
}

int32_t l2b_round_q8_host(float *data, uint64_t rows, uint64_t cols, uint64_t *n_changed) {
    if (!data || cols == 0 || cols > (1ull << 30)) return L2B_ERR_INVALID_ARG;
    for (uint64_t i = 0; i < rows * cols; ++i)   // refuse before anything is written
        if (!std::isfinite(data[i])) return L2B_ERR_INVALID_ARG;
    std::vector<unsigned char> rec((size_t)w_pitch<q8>((int)cols));
    const int so = q8_scale_off((int)cols);
    uint64_t changed = 0;
    for (uint64_t r = 0; r < rows; ++r) {
        float *w = data + r * cols;
        changed += (uint64_t)quantize_q8_row(w, cols, rec.data());
        for (uint64_t c = 0; c < cols; ++c) {
            float s;
            memcpy(&s, rec.data() + so + (c / Q8_GROUP) * 4, 4);
            w[c] = q8_dequant((int8_t)rec[c], s);
        }
    }
    if (n_changed) *n_changed = changed;
    return L2B_OK;
}

int32_t l2b_create_session(l2b_ctx **out, l2b_ctx *model) {
    if (!out || !model) { g_create_error = "NULL argument"; return L2B_ERR_INVALID_ARG; }
    *out = nullptr;
    if (model->world > 1) { g_create_error = "sessions need a single-GPU model (tensor parallel is not supported)"; return L2B_ERR_UNSUPPORTED; }
    l2b_ctx *ctx = new l2b_ctx();
    const int rc = create_session(ctx, model);
    if (rc) { destroy_rank(ctx); return rc; }
    *out = ctx;
    return L2B_OK;
}

void l2b_destroy(l2b_ctx *ctx) { destroy_all(ctx); }

int32_t l2b_reset(l2b_ctx *ctx) {
    if (!ctx) return L2B_ERR_INVALID_ARG;
    ctx->n_appended = 0;
    kv_release(ctx);
    return L2B_OK;
}

}  // extern "C" (a helper below)

// l2b_fork on a paged model: every destination gives up its pages, then shares src's full pages [0, n_pos/P)
// and gets a fresh page holding a copy of the rows of src's partial last page, [n_pos/P * P, n_pos).  The
// fresh pages are taken before any destination changes: a refused fork changes nothing.
int fork_paged(l2b_ctx *src, int32_t n_pos, l2b_ctx *const *dst, int32_t n_dst) {
    KvPool *pool = kv_pool(src);
    const int full = n_pos / KV_PAGE_ROWS, tail = n_pos % KV_PAGE_ROWS;
    L2B_CUDA(src, cudaSetDevice(src->device));
    std::vector<void *> fresh;
    for (int i = 0; tail && i < n_dst; ++i) {
        void *pg = nullptr;
        const int rc = kv_page_get(src, pool, &pg);
        if (rc) {
            for (void *f : fresh) kv_page_put(pool, f);
            return rc;
        }
        fresh.push_back(pg);
    }
    for (int i = 0; i < n_dst; ++i) {
        l2b_ctx *d = dst[i];
        for (int j = 0; j < d->n_pages; ++j) kv_drop(d, j);
        for (int j = 0; j < full; ++j) {
            d->pages[j] = src->pages[j];
            ++pool->refs[src->pages[j]];
            kv_tab_set(d, j, d->pages[j]);
        }
        if (tail) {
            d->pages[full] = fresh[i];
            kv_tab_set(d, full, fresh[i]);
        }
        d->n_appended = n_pos;
    }
    if (tail) {
        L2B_CUDA(src, cudaEventRecord(src->ev0, src->stream));
        int rc = kv_page_copy(src, src->pages[full], fresh.data(), n_dst, tail);
        if (rc) return rc;
        L2B_CUDA(src, cudaEventRecord(src->ev1, src->stream));
        L2B_CUDA(src, cudaEventSynchronize(src->ev1));
        L2B_CUDA(src, cudaEventElapsedTime(&src->last_ms, src->ev0, src->ev1));
    }
    for (int i = 0; i < n_dst; ++i) {
        const int rc = kv_tab_upload(dst[i]);
        if (rc) { src->err = dst[i]->err; return rc; }
    }
    return L2B_OK;
}

extern "C" {

// Everything is checked before anything launches.
int32_t l2b_fork(l2b_ctx *src, int32_t n_pos, l2b_ctx *const *dst, int32_t n_dst) {
    if (!src) { g_create_error = "src is NULL"; return L2B_ERR_INVALID_ARG; }
    if (!dst || n_dst < 1) return fail(src, L2B_ERR_INVALID_ARG, "dst is NULL or n_dst < 1");
    if (src->world > 1) return fail(src, L2B_ERR_UNSUPPORTED, "l2b_fork needs a single-GPU model (sessions are single-GPU only)");
    if (n_pos < 0) return fail(src, L2B_ERR_INVALID_ARG, "n_pos < 0");
    std::set<const l2b_ctx *> seen;
    for (int i = 0; i < n_dst; ++i) {
        const l2b_ctx *d = dst[i];
        if (!d) return fail(src, L2B_ERR_INVALID_ARG, "NULL destination");
        if (d == src) return fail(src, L2B_ERR_INVALID_ARG, "src among the destinations");
        if (!seen.insert(d).second) return fail(src, L2B_ERR_INVALID_ARG, "the same destination twice");
        if (d->weights != src->weights) return fail(src, L2B_ERR_INVALID_ARG, "a destination of another model");
    }
    if (n_pos > src->n_appended) return fail(src, L2B_ERR_STATE, "n_pos past the positions src has appended");
    src->last_ms = 0.0f;
    src->last_launches = 0;
    if (src->paged) return fork_paged(src, n_pos, dst, n_dst);
    if (n_pos > 0) {
        // No wait across streams: every call of this library ends in a synchronise, so neither src's
        // stream nor any destination's holds work when l2b_fork is entered, and the copy is synchronised
        // below before any destination can run again.
        cudaStream_t st = src->stream;
        L2B_CUDA(src, cudaSetDevice(src->device));
        L2B_CUDA(src, cudaEventRecord(src->ev0, st));
        std::vector<std::pair<void *, void *>> d;
        for (int i = 0; i < n_dst; ++i) d.emplace_back(dst[i]->kcache, dst[i]->vcache);
        const int rc = kv_fork_launch(src, src->kcache, src->vcache, (long long)n_pos * src->kv_loc,
                                      (long long)src->cfg.seq_len * src->kv_loc, d);
        if (rc) return rc;
        L2B_CUDA(src, cudaEventRecord(src->ev1, st));
        L2B_CUDA(src, cudaEventSynchronize(src->ev1));
        L2B_CUDA(src, cudaEventElapsedTime(&src->last_ms, src->ev0, src->ev1));
    }
    for (int i = 0; i < n_dst; ++i) dst[i]->n_appended = n_pos;
    return L2B_OK;
}

float *l2b_logits_buffer(l2b_ctx *ctx) { return ctx ? ctx->h_logits : nullptr; }

int32_t l2b_forward_pinned(l2b_ctx *ctx, int32_t token, int32_t pos, const float **logits) {
    int rc = check_step_args(ctx, token, pos);
    if (rc) return rc;
    if (!logits) return fail(ctx, L2B_ERR_INVALID_ARG, "logits is NULL");
    rc = run_step(ctx, token, pos, G_LOGITS, 1.0f, 0.0f);
    if (rc) return rc;
    *logits = ctx->h_logits;
    return L2B_OK;
}

int32_t l2b_forward(l2b_ctx *ctx, int32_t token, int32_t pos, float *host_logits) {
    int rc = check_step_args(ctx, token, pos);
    if (rc) return rc;
    if (!host_logits) return fail(ctx, L2B_ERR_INVALID_ARG, "host_logits is NULL");
    rc = run_step(ctx, token, pos, G_LOGITS, 1.0f, 0.0f);
    if (rc) return rc;
    // state.logits of the reference is one long-lived buffer (src/main.zig:149).  A host that
    // adopted l2b_logits_buffer() as that buffer gets the logits without a second copy; any other
    // destination gets one streaming memcpy from the pinned landing buffer.
    if (host_logits != ctx->h_logits)
        memcpy(host_logits, ctx->h_logits, (size_t)ctx->cfg.vocab_size * sizeof(float));
    return L2B_OK;
}

int32_t l2b_forward_argmax(l2b_ctx *ctx, int32_t token, int32_t pos, int32_t *next) {
    int rc = check_step_args(ctx, token, pos);
    if (rc) return rc;
    if (!next) return fail(ctx, L2B_ERR_INVALID_ARG, "next is NULL");
    rc = run_step(ctx, token, pos, G_ARGMAX_ONE, 1.0f, 0.0f);
    if (rc) return rc;
    *next = ctx->h_ints[0];
    return L2B_OK;
}

int32_t l2b_forward_sample(l2b_ctx *ctx, int32_t token, int32_t pos, float temperature, float top_p,
                           float *host_probs, l2b_prob_index *cand, int32_t cand_cap, int32_t *n_cand) {
    int rc = check_step_args(ctx, token, pos);
    if (rc) return rc;
    if (!(temperature > 0.0f)) return fail(ctx, L2B_ERR_INVALID_ARG, "temperature must be > 0 (use l2b_forward_argmax for 0)");
    if (top_p < 0.0f || top_p > 1.0f) return fail(ctx, L2B_ERR_INVALID_ARG, "top_p must be in [0, 1]");
    // like l2b_op_sample_prep: the top-p cutoff (1-p)/(n-1) has no meaning for a single entry
    if (ctx->cfg.vocab_size < 2) return fail(ctx, L2B_ERR_INVALID_ARG, "sampling needs vocab_size >= 2");
    const bool filter = (top_p != 0.0f && top_p != 1.0f);            // :1009
    if (filter && (!cand || !n_cand || cand_cap <= 0)) return fail(ctx, L2B_ERR_INVALID_ARG, "candidate buffer missing");
    rc = run_step(ctx, token, pos, G_SAMPLE, temperature, filter ? top_p : -1.0f);
    if (rc) return rc;
    copy_step_sample_out(ctx, filter, host_probs, cand, cand_cap, n_cand);
    return L2B_OK;
}

}  // extern "C" (templates below)

// ---- batched prompt prefill (prefill_gemm_kernel in l2b_device.cuh) -----------------------------
// the batched-prefill kernel of NB vectors for the context's formats (no EPI_XCHG: single GPU only)
template <int NB>
gemv_fn pf_pick(const l2b_ctx *ctx, int epi) {
    return with_w(ctx->wfmt, [&](auto w) {
        using W = typename decltype(w)::type;
        return pick_epi<W, false>(ctx, epi, [](auto e, auto kv) { return (gemv_fn)prefill_gemm_kernel<decltype(e)::value, NB, W, typename decltype(kv)::type>; });
    });
}
constexpr size_t kPfSmemBudget = 227 * 1024 - 8192;   // the prefill kernels keep ~6.5 KB of static shared memory

// can this context prefill PF_MAXB positions per weight pass?  Single GPU, flash attention, and all
// four per-layer GEMVs bandwidth-bound shapes of the TMA-ring kernel; otherwise l2b_prefill runs the
// positions one by one on the device (same results, weights streamed once per position).  The batched
// step (l2b_forward_batch) makes the same choice on its first session; its classifier's dim-wide
// inputs fit wherever qkv's do.
static int pf_prepare(l2b_ctx *ctx) {
    if (ctx->pf_ready) return L2B_OK;
    ctx->pf_ready = true;
    const char *env = getenv("L2B_PREFILL_BATCH");
    if (env && env[0] == '0') return L2B_OK;
    const uint64_t dim = ctx->dim, hid = ctx->hid_loc, q = ctx->q_loc;
    size_t smem = 0;
    const bool shapes_ok = ctx->world == 1 && !ctx->leader && dim >= (uint64_t)ctx->big_min_n && hid >= (uint64_t)ctx->big_min_n &&
                           dim <= TMA_MAXV * TMA_PRO_THREADS * 4 && ctx->gemv8_min_bytes >= 0 &&
                           dim * dim * 4 >= (uint64_t)ctx->gemv8_min_bytes && ctx->attn_flash &&
                           pick_attention(ctx->head_size, true, &smem) != attention_kernel<float> &&
                           pf_ring_stages(kPfSmemBudget, PF_MAXB * dim * 4) >= 2 &&
                           pf_ring_stages(kPfSmemBudget, 2 * hid * 4) >= 2;
    if (!shapes_ok) return L2B_OK;
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc;
    if ((rc = dev_alloc(ctx, &ctx->pf_x, PF_MAXB * dim))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->pf_q, PF_MAXB * q))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->pf_xb, PF_MAXB * q))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->pf_hb, PF_MAXB * hid))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->pf_logits, (size_t)PF_MAXB * ctx->vocab_loc))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->pf_amax, (size_t)PF_MAXB))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->pf_part_o, (size_t)PF_MAXB * ctx->heads_loc * ctx->nsplit * ctx->head_size))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->pf_part_ml, (size_t)PF_MAXB * ctx->heads_loc * ctx->nsplit * 2))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->pf_counters, (size_t)PF_MAXB * ctx->heads_loc))) return rc;
    L2B_CUDA(ctx, cudaMemsetAsync(ctx->pf_counters, 0, (size_t)PF_MAXB * ctx->heads_loc * sizeof(unsigned int), ctx->stream));
    for (int epi : {(int)EPI_QKV, (int)EPI_SILU, (int)EPI_RESID, (int)EPI_STORE, (int)EPI_ARGMAX}) {
        L2B_CUDA(ctx, cudaFuncSetAttribute(pf_pick<PF_MAXB>(ctx, epi), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPfSmemBudget));
        L2B_CUDA(ctx, cudaFuncSetAttribute(pf_pick<2>(ctx, epi), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPfSmemBudget));
    }
    ctx->pf_ok = true;
    return L2B_OK;
}

template <int NB>
static int pf_launch(l2b_ctx *ctx, int epi, GemvParams p, cudaStream_t st) {
    const size_t xbytes = (size_t)NB * p.n * 4;
    const int nstage = pf_ring_stages(kPfSmemBudget, xbytes);
    // the same ring bytes in the format's stages: 32 KB fp32, 16 KB bf16, 17 KB q8
    p.nstage = with_w(ctx->wfmt, [nstage](auto w) { return pf_stages<typename decltype(w)::type>(nstage); });
    int grid = ctx->num_sms;
    const int npairs = (p.total_rows + 1) / 2;
    if (grid > npairs) grid = npairs;
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(grid);
    lc.blockDim = dim3(TMA_THREADS);
    lc.dynamicSmemBytes = (size_t)nstage * TMA_STAGE_FLOATS * 4 + xbytes;
    // hard invariant, whatever pf_prepare decided: a ring kernel never launches with fewer than 2 stages
    if (nstage < 2 || lc.dynamicSmemBytes > kPfSmemBudget)
        return fail(ctx, L2B_ERR_UNSUPPORTED, "batched prefill: TMA ring of fewer than 2 stages or past the shared-memory budget");
    lc.stream = st;
    cudaLaunchAttribute at[1] = {pdl_attr()};
    lc.attrs = at;
    lc.numAttrs = ctx->use_pdl ? 1 : 0;
    const gemv_fn fn = pf_pick<NB>(ctx, epi);
    if (!fn) return fail(ctx, L2B_ERR_UNSUPPORTED, "batched prefill: no kernel for this epilogue");
    L2B_CUDA(ctx, cudaLaunchKernelEx(&lc, fn, p));
    ++ctx->last_launches;
    return L2B_OK;
}

// nb <= PF_MAXB vectors through every layer in one pass over the weights, on ctx's stream and batch
// buffers: vector b enters as the embedding row of d_tokens[b] and runs at position pos[b] on the KV
// cache of kv[b] (a prompt: one context at consecutive positions; the batched step: one session per
// vector).  Its x is left in ctx->pf_x[b].  d_skip (device, or nullptr): vector b appends no KV row
// when d_skip[b] is set (a stopped session of the batched generation loop).
static int batched_layers(l2b_ctx *ctx, l2b_ctx *const *kv, const int *pos, int nb, const int *d_tokens,
                          const int *d_skip) {
    const int dim = ctx->dim;
    cudaStream_t st = ctx->stream;
    for (int l = 0; l < ctx->cfg.n_layers; ++l) {
        LayerGemvs g = layer_gemvs(ctx, l);
        AttnBatch zb{};
        for (int b = 0; b < nb; ++b) {
            g.qkv.pos_b[b] = zb.pos[b] = pos[b];
            g.qkv.kcache_b[b] = kv_layer(kv[b], kv[b]->kcache, l);
            g.qkv.vcache_b[b] = kv_layer(kv[b], kv[b]->vcache, l);
            zb.kcache[b] = g.qkv.kcache_b[b];
            zb.vcache[b] = g.qkv.vcache_b[b];
        }
        // ---- rmsnorm + q,k,v + RoPE + KV append for nb vectors (:305-358)
        g.qkv.nb = nb;
        g.qkv.skip_b = d_skip;
        g.qkv.x_in = ctx->pf_x;
        if (l == 0) { g.qkv.emb = ctx->emb; g.qkv.tokens = d_tokens; g.qkv.x_out = ctx->pf_x; }
        g.qkv.out0 = ctx->pf_q;
        int rc = pf_launch<PF_MAXB>(ctx, EPI_QKV, g.qkv, st);
        if (rc) return rc;
        // ---- attention of the nb queries (:361-389); query z sees positions 0 .. pos[z] of its cache
        rc = launch_attention(ctx, l, st, ctx->pf_q, ctx->pf_xb, ctx->pf_part_o, ctx->pf_part_ml, ctx->pf_counters,
                              &zb, ctx->q_loc, nb);
        if (rc) return rc;
        // ---- wo + residual (:392-395)
        g.wo.nb = nb;
        g.wo.x_in = ctx->pf_xb;
        g.wo.out0 = ctx->pf_x;
        rc = pf_launch<PF_MAXB>(ctx, EPI_RESID, g.wo, st);
        if (rc) return rc;
        // ---- rmsnorm + w1,w3 + SiLU*mul (:398-416)
        g.w13.nb = nb;
        g.w13.x_in = ctx->pf_x;
        g.w13.out0 = ctx->pf_hb;
        rc = pf_launch<PF_MAXB>(ctx, EPI_SILU, g.w13, st);
        if (rc) return rc;
        // ---- w2 + residual (:419-422); hidden-sized inputs: two vectors per pass (shared memory)
        for (int b = 0; b < nb; b += 2) {
            GemvParams d = g.w2;
            d.nb = nb - b < 2 ? nb - b : 2;
            d.x_in = ctx->pf_hb + (size_t)b * ctx->hid_loc;
            d.out0 = ctx->pf_x + (size_t)b * dim;
            rc = pf_launch<2>(ctx, EPI_RESID, d, st);
            if (rc) return rc;
        }
    }
    return L2B_OK;
}

static int batched_classifier(l2b_ctx *ctx, int nb, bool argmax);
static int launch_logprob_batch(l2b_ctx *ctx, int nb, int done);

// a per-call device buffer of ctx (call_ints, call_cand): at least `count` entries, grown on demand; the
// current device is ctx's
template <typename T>
static int call_buf_reserve(l2b_ctx *ctx, T *&buf, size_t &cap, size_t count) {
    if (cap >= count) return L2B_OK;
    if (buf) {
        L2B_CUDA(ctx, cudaFree(buf));
        ctx->owned.erase(std::find(ctx->owned.begin(), ctx->owned.end(), (void *)buf));
        buf = nullptr;
        cap = 0;
    }
    const int rc = dev_alloc(ctx, &buf, count);
    if (rc) { cudaGetLastError(); return rc; }
    cap = count;
    return L2B_OK;
}

// The prologue of a batched call on ctx (the current device): the call's `count` ints, its tokens among
// them, to call_ints in one copy (from pageable memory: staged before this returns), the argmax keys
// zeroed, the control block with DONE = 0 (for the attention kernel, and until an early exit raises
// it), then ev0.  Everything enqueued from here to batched_end is the call's timed work.
static int batched_begin(l2b_ctx *ctx, const int32_t *ints, size_t count, int token0, int pos0) {
    cudaStream_t st = ctx->stream;
    int rc = call_buf_reserve(ctx, ctx->call_ints, ctx->call_ints_cap, count);
    if (rc) return rc;
    L2B_CUDA(ctx, cudaMemcpyAsync(ctx->call_ints, ints, count * sizeof(int), cudaMemcpyHostToDevice, st));
    L2B_CUDA(ctx, cudaMemsetAsync(ctx->pf_amax, 0, PF_MAXB * sizeof(unsigned long long), st));
    fill_ctl(ctx, token0, pos0, 0, 1.0f, -1.0f);
    L2B_CUDA(ctx, cudaMemcpyAsync(ctx->ctl, ctx->h_ctl, CTL_HOST_WORDS * sizeof(int), cudaMemcpyHostToDevice, st));
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev0, st));
    ctx->last_launches = 0;
    return L2B_OK;
}

// The epilogue: with back, `count` result ints from call_ints + from to back; then ev1, one synchronise,
// and the call's device time in last_ms.
static int batched_end(l2b_ctx *ctx, int *back, size_t from, size_t count) {
    cudaStream_t st = ctx->stream;
    if (back) L2B_CUDA(ctx, cudaMemcpyAsync(back, ctx->call_ints + from, count * sizeof(int), cudaMemcpyDeviceToHost, st));
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev1, st));
    L2B_CUDA(ctx, cudaStreamSynchronize(st));
    L2B_CUDA(ctx, cudaGetLastError());
    L2B_CUDA(ctx, cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
    return L2B_OK;
}

// The vectors of n runs laid back to back: run i is n_tok[i] vectors (n_tok == nullptr: one each) on
// session s[i] from pos[i] on, and vector v runs at pos[v] on the cache of kv[v], entry j[v] of run run[v].
struct RunVectors {
    std::vector<l2b_ctx *> kv;
    std::vector<int> pos, run, j;
};
static RunVectors expand_runs(l2b_ctx *const *s, int n, const int32_t *n_tok, const int32_t *pos) {
    RunVectors r;
    for (int i = 0; i < n; ++i)
        for (int j = 0, len = n_tok ? n_tok[i] : 1; j < len; ++j) {
            r.kv.push_back(s[i]);
            r.pos.push_back(pos[i] + j);
            r.run.push_back(i);
            r.j.push_back(j);
        }
    return r;
}

// n_tokens positions starting at pos0, PF_MAXB per pass over the weights; KV cache filled.  Without
// score no logits; with score (l2b_score: tokens holds n_tokens + 1 entries, all staged) each group then
// runs the argmax classifier and logprob_batch_kernel, which leaves position i's log-probability of
// tokens[i + 1] and its greedy token in score_lp[i] and score_greedy[i].
static int prefill_batched(l2b_ctx *ctx, const int32_t *tokens, int n_tokens, int pos0, bool score = false) {
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    const RunVectors r = expand_runs(&ctx, 1, &n_tokens, &pos0);
    int rc = batched_begin(ctx, tokens, (size_t)n_tokens + (score ? 1 : 0), tokens[0], pos0);
    if (rc) return rc;
    for (int done = 0; done < n_tokens; done += PF_MAXB) {
        const int nb = n_tokens - done < PF_MAXB ? n_tokens - done : PF_MAXB;
        rc = batched_layers(ctx, r.kv.data() + done, r.pos.data() + done, nb, ctx->call_ints + done, nullptr);
        if (rc) return rc;
        if (score) {
            rc = batched_classifier(ctx, nb, true);
            if (rc) return rc;
            rc = launch_logprob_batch(ctx, nb, done);
            if (rc) return rc;
        }
    }
    rc = batched_end(ctx, nullptr, 0, 0);
    if (rc) return rc;
    if (pos0 + n_tokens > ctx->n_appended) ctx->n_appended = pos0 + n_tokens;
    return L2B_OK;
}

// final rmsnorm + classifier (:426-429) of the nb vectors in ctx->pf_x: logits to pf_logits, and with
// argmax one packed key per vector added into pf_amax (zero before the launch)
static int batched_classifier(l2b_ctx *ctx, int nb, bool argmax) {
    GemvParams k{};
    k.ctl = ctx->ctl;
    k.n = ctx->dim;
    k.nb = nb;
    k.x_in = ctx->pf_x;
    k.gamma = ctx->rms_final;
    k.w0 = ctx->wcls;
    k.total_rows = ctx->cfg.vocab_size; k.rows0 = ctx->cfg.vocab_size;
    k.out0 = ctx->pf_logits;
    k.amax = ctx->pf_amax;
    return pf_launch<PF_MAXB>(ctx, argmax ? EPI_ARGMAX : EPI_STORE, k, ctx->stream);
}

// logprob_batch_kernel over the nb logits rows of a group in pf_logits: positions done .. done+nb-1 of a
// score, their targets the staged tokens at call_ints + 1 + done, their results to score_lp / score_greedy + done
static int launch_logprob_batch(l2b_ctx *ctx, int nb, int done) {
    LogprobBatchParams p{};
    p.ctl = ctx->ctl;
    p.logits = ctx->pf_logits;
    p.n = ctx->cfg.vocab_size;
    p.targets = ctx->call_ints + 1 + done;
    p.amax = ctx->pf_amax;
    p.lp = ctx->score_lp + done;
    p.greedy = ctx->score_greedy + done;
    void *args[] = {&p};
    return launch_small(ctx, (const void *)logprob_batch_kernel, dim3(nb), dim3(LOGPROB_THREADS), args, ctx->stream, true);
}

// Everything a batched call checks, before anything is launched: a refused call changes no session.
// ragged: session i runs n_tok[i] tokens (tokens holds the runs back to back) at pos[i] ..; otherwise
// one token each and n_tok is ignored.
static int check_batch_args(l2b_ctx *const *s, int32_t n, const int32_t *tokens, const int32_t *pos,
                            bool ragged = false, const int32_t *n_tok = nullptr) {
    if (!s || n < 1 || !s[0]) { g_create_error = "sessions is NULL, n < 1 or sessions[0] is NULL"; return L2B_ERR_INVALID_ARG; }
    l2b_ctx *s0 = s[0];
    if (!tokens || !pos) return fail(s0, L2B_ERR_INVALID_ARG, "tokens or pos is NULL");
    if (ragged && !n_tok) return fail(s0, L2B_ERR_INVALID_ARG, "n_tokens is NULL");
    std::set<const l2b_ctx *> seen;
    int64_t off = 0;                                     // the run's first entry in tokens
    for (int i = 0; i < n; ++i) {
        const l2b_ctx *c = s[i];
        if (!c) return fail(s0, L2B_ERR_INVALID_ARG, "NULL session");
        if (!seen.insert(c).second) return fail(s0, L2B_ERR_INVALID_ARG, "the same session twice in one batch");
        if (c->weights != s0->weights) return fail(s0, L2B_ERR_INVALID_ARG, "sessions of different models");
        const int64_t len = ragged ? n_tok[i] : 1;
        if (len < 1) return fail(s0, L2B_ERR_INVALID_ARG, "n_tokens < 1");
        if (pos[i] < 0 || pos[i] >= c->cfg.seq_len) return fail(s0, L2B_ERR_INVALID_ARG, "pos out of range");
        if (pos[i] + len > c->cfg.seq_len) return fail(s0, L2B_ERR_INVALID_ARG, "run past seq_len");
        if (off + len > INT32_MAX) return fail(s0, L2B_ERR_INVALID_ARG, "total token count overflows int32");
        for (int64_t j = off; j < off + len; ++j)   // the run's tokens are read only once its length is known sound
            if (tokens[j] < 0 || tokens[j] >= c->cfg.vocab_size) return fail(s0, L2B_ERR_INVALID_ARG, "token out of range");
        off += len;
    }
    for (int i = 0; i < n; ++i)
        if (pos[i] > s[i]->n_appended) return fail(s0, L2B_ERR_STATE, "pos skips ahead of a session's KV cache");
    return L2B_OK;
}

// sample_prep_batch_kernel over the nb logits rows of a group in pf_logits, in place; row b with
// temperature[b] and top_p[b] (< 0: no filter), its kCandCap candidates to cand[b] and their count to n_cand[b]
static int launch_sample_prep_batch(l2b_ctx *ctx, int nb, const float *temperature, const float *top_p,
                                    ProbIndex *const *cand, int *const *n_cand) {
    SamplePrepBatchParams p{};
    p.ctl = ctx->ctl;
    p.logits = ctx->pf_logits;
    p.n = p.stride = ctx->cfg.vocab_size;
    p.cand_cap = kCandCap;
    for (int b = 0; b < nb; ++b) {
        p.temperature[b] = temperature[b];
        p.top_p[b] = top_p[b];
        p.cand[b] = cand[b];
        p.n_cand[b] = n_cand[b];
    }
    void *args[] = {&p};
    return launch_small(ctx, (const void *)sample_prep_batch_kernel, dim3(nb), dim3(SAMP_THREADS), args, ctx->stream, true);
}

// One run of each of n validated sessions: session i runs its n_tok[i] tokens (tokens holds the runs
// back to back) at positions pos[i] .. pos[i] + n_tok[i] - 1; n_tok == nullptr: one token each (the
// batched step).  Only a run's last position has an output.
// Where l2b_prefill would batch (pf_prepare on the first session), the runs' positions, concatenated in
// session order, go PF_MAXB per pass over the weights on the first session's stream and batch buffers,
// each vector on its own session's cache at its own position (a run may straddle groups).  A group
// holding some run's last vector then runs the batched classifier, and each such vector's x and logits
// are copied to its session's own buffers (xb, hb and q are not written); a vector that ends no run
// writes nothing into any session.  Otherwise each session runs l2b_prefill of its run but the last
// token (no logits), and then its own step of the last token.  mode: MODE_LOGITS leaves each session's
// logits in its h_logits, MODE_ARGMAX the next token in its h_ints[0], and MODE_SAMPLE (temperature[i],
// top_p[i] < 0: no filter) its probabilities in h_logits, candidates in h_cand and their count in
// h_ints[2], as l2b_forward_sample's step does.  The call's time and launches on s[0].
static int step_sessions(l2b_ctx *const *s, int n, const int32_t *n_tok, const int32_t *tokens, const int32_t *pos,
                         StepMode mode, const float *temperature = nullptr, const float *top_p = nullptr) {
    l2b_ctx *ctx = s[0];
    const bool argmax = (mode == MODE_ARGMAX), sample = (mode == MODE_SAMPLE);
    std::vector<KvRange> ranges;
    for (int i = 0; i < n; ++i) ranges.push_back(KvRange{s[i], pos[i], pos[i] + (n_tok ? n_tok[i] : 1)});
    KvCall kv;
    int rc = kv.reserve(ctx, ranges);
    if (rc) return rc;
    rc = pf_prepare(ctx);
    if (rc) return rc;
    // the vectors: vector v runs token tokens[v]; last(v): the session it ends, or -1
    const RunVectors r = expand_runs(s, n, n_tok, pos);
    const int total = (int)r.kv.size();
    auto last = [&](int v) { return r.j[v] == (n_tok ? n_tok[r.run[v]] : 1) - 1 ? r.run[v] : -1; };
    cudaStream_t st = ctx->stream;
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->pf_ok) {
        // a run's leading tokens first, session by session; each prefill times itself on its session's events
        float pre_ms = 0.0f;
        int launches = 0;
        for (int v = 0, i = 0; v < total; ++v) {
            if (last(v) < 0) continue;
            const int len = n_tok ? n_tok[i] : 1;
            if (len > 1) {
                rc = l2b_prefill(s[i], tokens + v - (len - 1), len - 1, pos[i], nullptr);
                if (rc) { ctx->err = s[i]->err; return rc; }
                pre_ms += s[i]->last_ms;
                launches += s[i]->last_launches;
            }
            ++i;
        }
        L2B_CUDA(ctx, cudaEventRecord(ctx->ev0, st));
        for (int v = 0; v < total; ++v) {
            const int i = last(v);
            if (i < 0) continue;
            rc = sample ? run_step(s[i], tokens[v], r.pos[v], G_SAMPLE, temperature[i], top_p[i])
                        : run_step(s[i], tokens[v], r.pos[v], argmax ? G_ARGMAX_ONE : G_LOGITS, 1.0f, 0.0f);
            if (rc) { ctx->err = s[i]->err; return rc; }
            launches += s[i]->last_launches;
        }
        // every step above ended in a synchronise: ev0 .. ev1 spans them all
        L2B_CUDA(ctx, cudaEventRecord(ctx->ev1, s[n - 1]->stream));
        L2B_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
        L2B_CUDA(ctx, cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
        ctx->last_ms += pre_ms;
        ctx->last_launches = launches;
        return L2B_OK;
    }
    const int dim = ctx->dim, V = ctx->cfg.vocab_size;
    rc = batched_begin(ctx, tokens, total, tokens[0], pos[0]);
    if (rc) return rc;
    for (int g = 0; g < total; g += PF_MAXB) {
        const int nb = total - g < PF_MAXB ? total - g : PF_MAXB;
        rc = batched_layers(ctx, r.kv.data() + g, r.pos.data() + g, nb, ctx->call_ints + g, nullptr);
        if (rc) return rc;
        // the group's vectors that end a run: row[k] in the group, of session ends[k]
        int row[PF_MAXB], nl = 0;
        l2b_ctx *ends[PF_MAXB];
        float lt[PF_MAXB], lp[PF_MAXB];
        ProbIndex *lc[PF_MAXB];
        int *ln[PF_MAXB];
        for (int b = 0; b < nb; ++b) {
            const int i = last(g + b);
            if (i < 0) continue;
            row[nl] = b;
            ends[nl] = s[i];
            if (sample) { lt[nl] = temperature[i]; lp[nl] = top_p[i]; lc[nl] = s[i]->cand; ln[nl] = s[i]->n_cand; }
            ++nl;
        }
        if (nl == 0) continue;
        if (argmax) L2B_CUDA(ctx, cudaMemsetAsync(ctx->pf_amax, 0, PF_MAXB * sizeof(unsigned long long), st));
        rc = batched_classifier(ctx, nb, argmax);
        if (rc) return rc;
        if (sample) {
            // the sampler works on the first nl rows: the last rows move to the front, in row order (row k
            // receives row[k] >= k, so every row is read before a copy writes over it); then logits ->
            // probabilities in place, candidates to each session's own buffers
            for (int k = 0; k < nl; ++k)
                if (row[k] != k)
                    L2B_CUDA(ctx, cudaMemcpyAsync(ctx->pf_logits + (size_t)k * V, ctx->pf_logits + (size_t)row[k] * V,
                                                  V * sizeof(float), cudaMemcpyDeviceToDevice, st));
            rc = launch_sample_prep_batch(ctx, nl, lt, lp, lc, ln);
            if (rc) return rc;
        }
        for (int k = 0; k < nl; ++k) {
            l2b_ctx *c = ends[k];
            const int b = row[k];
            const float *lg = ctx->pf_logits + (size_t)(sample ? k : b) * V;
            L2B_CUDA(ctx, cudaMemcpyAsync(c->X, ctx->pf_x + (size_t)b * dim, dim * sizeof(float), cudaMemcpyDeviceToDevice, st));
            L2B_CUDA(ctx, cudaMemcpyAsync(c->logits, lg, V * sizeof(float), cudaMemcpyDeviceToDevice, st));
            if (argmax)   // the key's low word (little-endian: its first 4 bytes) is 0xFFFFFFFF - index
                L2B_CUDA(ctx, cudaMemcpyAsync(c->h_ints, ctx->pf_amax + b, sizeof(int), cudaMemcpyDeviceToHost, st));
            else
                L2B_CUDA(ctx, cudaMemcpyAsync(c->h_logits, lg, V * sizeof(float), cudaMemcpyDeviceToHost, st));
            if (sample) {   // as the single step's G_SAMPLE graph copies them
                L2B_CUDA(ctx, cudaMemcpyAsync(c->h_cand, c->cand, (size_t)kCandCap * sizeof(ProbIndex), cudaMemcpyDeviceToHost, st));
                L2B_CUDA(ctx, cudaMemcpyAsync(c->h_ints + 2, c->n_cand, sizeof(int), cudaMemcpyDeviceToHost, st));
            }
        }
    }
    rc = batched_end(ctx, nullptr, 0, 0);
    if (rc) return rc;
    for (int i = 0; i < n; ++i) {
        l2b_ctx *c = s[i];
        const int end = pos[i] + (n_tok ? n_tok[i] : 1);
        c->final_X = c->X;
        if (argmax) c->h_ints[0] = (int)(0xFFFFFFFFu - (uint32_t)c->h_ints[0]);
        if (end > c->n_appended) c->n_appended = end;
    }
    return L2B_OK;
}

extern "C" {

// One on-device loop of one context: n_steps replays of a device-loop graph (G_ARGMAX_LOOP or
// G_PREFILL_LOOP) starting at (token, pos).  The loops of one call are the ranks of an in-process group
// (all but the lead are not sinks: their tokens are the lead's) or several sessions (all sinks).
struct DeviceLoop {
    l2b_ctx *c;
    int token, pos, n_steps;
    const int32_t *forced;   // n_steps entries, -1 = free-running, or nullptr
    bool sink;               // its tokens, n_done and appended count are read back
    int launches = 0, done = 0;
};

// The enqueue half: every loop's inputs, then its replays, then the copies of its results; nothing is
// synchronised.  Timing events go on the lead's stream (loops[0]); loops on other streams of the lead's
// device are bracketed by them too.
static int enqueue_device_loops(std::vector<DeviceLoop> &loops, int which, int stop_on_bos) {
    l2b_ctx *ctx = loops[0].c;
    int rc;
    for (DeviceLoop &d : loops) {
        l2b_ctx *c = d.c;
        L2B_CUDA(ctx, cudaSetDevice(c->device));
        // forced tokens (prompt forcing, :999-1000); -1 = free-running
        for (int i = 0; i < d.n_steps; ++i) c->h_gen[i] = d.forced ? d.forced[i] : -1;
        L2B_CUDA(ctx, cudaMemcpyAsync(c->gen_forced, c->h_gen, (size_t)d.n_steps * sizeof(int),
                                      cudaMemcpyHostToDevice, c->stream));
        L2B_CUDA(ctx, cudaMemsetAsync(c->gen_ndone, 0, sizeof(int), c->stream));
        L2B_CUDA(ctx, cudaMemsetAsync(c->amax, 0, sizeof(unsigned long long), c->stream));
        fill_ctl(c, d.token, d.pos, stop_on_bos ? 1 : 0, 1.0f, -1.0f);
        if (c == ctx) L2B_CUDA(ctx, cudaEventRecord(c->ev0, c->stream));
        L2B_CUDA(ctx, cudaMemcpyAsync(c->ctl, c->h_ctl, CTL_HOST_WORDS * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    }
    for (DeviceLoop &d : loops)
        if (d.c->device == ctx->device && d.c->stream != ctx->stream)
            L2B_CUDA(ctx, cudaStreamWaitEvent(d.c->stream, ctx->ev0, 0));
    // the whole step depends on (token,pos) only through ctl, which advance_kernel updates, so the
    // same graph is replayed back to back with no host round trip; with several loops the launches
    // are interleaved so that no stream's queue runs dry while another's is being filled
    int n_max = 0;
    for (const DeviceLoop &d : loops) n_max = d.n_steps > n_max ? d.n_steps : n_max;
    for (int i = 0; i < n_max; ++i) {
        for (DeviceLoop &d : loops) {
            l2b_ctx *c = d.c;
            if (i >= d.n_steps) continue;
            if (loops.size() > 1) L2B_CUDA(ctx, cudaSetDevice(c->device));
            if (c->use_graphs) {
                L2B_CUDA(ctx, cudaGraphLaunch(c->graphs[which], c->stream));
                // G_LOGITS' count, minus the classifier (prefill), plus advance_kernel and logprob_kernel (score)
                d.launches += c->launches_per_step + (which == G_PREFILL_LOOP ? 0 : which == G_SCORE_LOOP ? 2 : 1);
            } else {
                c->last_launches = 0;
                rc = enqueue_call(c, c->stream, which);
                if (rc) { ctx->err = c->err; return rc; }
                d.launches += c->last_launches;
            }
        }
    }
    // the lead last: its end event follows every other stream of its device
    for (size_t k = loops.size(); k-- > 0;) {
        l2b_ctx *c = loops[k].c;
        L2B_CUDA(ctx, cudaSetDevice(c->device));
        if (loops[k].sink) {
            L2B_CUDA(ctx, cudaMemcpyAsync(c->h_gen, c->gen_out, (size_t)loops[k].n_steps * sizeof(int),
                                          cudaMemcpyDeviceToHost, c->stream));
            L2B_CUDA(ctx, cudaMemcpyAsync(c->h_ints + 1, c->gen_ndone, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        }
        L2B_CUDA(ctx, cudaMemcpyAsync(c->h_ctl + CTL_WORDS, c->ctl, CTL_WORDS * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        if (c == ctx) {
            L2B_CUDA(ctx, cudaEventRecord(c->ev1, c->stream));
        } else if (c->device == ctx->device && c->stream != ctx->stream) {
            L2B_CUDA(ctx, cudaEventRecord(c->ev1, c->stream));
            L2B_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, c->ev1, 0));
        }
    }
    return L2B_OK;
}

// The finish half: one synchronise of every loop's stream, then each sink's steps done (its tokens in
// h_gen) and appended count; the call's device time on the lead.
static int finish_device_loops(std::vector<DeviceLoop> &loops) {
    l2b_ctx *ctx = loops[0].c;
    std::vector<l2b_ctx *> cs;
    for (const DeviceLoop &d : loops) cs.push_back(d.c);
    int rc = finish_call(cs.data(), cs.size());
    if (rc) return rc;
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    L2B_CUDA(ctx, cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
    for (DeviceLoop &d : loops) {
        if (!d.sink) continue;
        d.done = d.c->h_ints[1];
        if (d.pos + d.done > d.c->n_appended) d.c->n_appended = d.pos + d.done;
    }
    return L2B_OK;
}

// n_steps replays of a device-loop graph (G_ARGMAX_LOOP or G_PREFILL_LOOP) on every rank of ctx
static int run_device_loop(l2b_ctx *ctx, int which, int token, int pos, int n_steps, const int32_t *forced,
                           int stop_on_bos, int *done_out) {
    std::vector<DeviceLoop> loops;
    for (l2b_ctx *c : locals(ctx)) loops.push_back(DeviceLoop{c, token, pos, n_steps, forced, c == ctx});
    int rc = enqueue_device_loops(loops, which, stop_on_bos);
    if (rc) return rc;
    rc = finish_device_loops(loops);
    if (rc) return rc;
    *done_out = loops[0].done;
    ctx->last_launches = loops[0].launches;
    return L2B_OK;
}

// forced tokens a generate call reads: -1 (free-running) or a token of the vocabulary, which the next
// step embeds; anything else is refused before anything runs
static int check_forced(l2b_ctx *ctx, const int32_t *forced, int count) {
    if (!forced) return L2B_OK;
    for (int i = 0; i < count; ++i)
        if (forced[i] < -1 || forced[i] >= ctx->cfg.vocab_size) return fail(ctx, L2B_ERR_INVALID_ARG, "forced token out of range");
    return L2B_OK;
}

int32_t l2b_generate_argmax(l2b_ctx *ctx, int32_t token, int32_t pos, int32_t n_steps,
                            const int32_t *forced, int32_t stop_on_bos, int32_t *out_next,
                            int32_t *n_done) {
    int rc = check_step_args(ctx, token, pos);
    if (rc) return rc;
    if (!out_next || !n_done || n_steps < 0) return fail(ctx, L2B_ERR_INVALID_ARG, "bad generate arguments");
    if (n_steps > ctx->cfg.seq_len - pos) n_steps = ctx->cfg.seq_len - pos;   // :992-993
    rc = check_forced(ctx, forced, n_steps);
    if (rc) return rc;
    *n_done = 0;
    if (n_steps == 0) return L2B_OK;
    KvCall kv;
    rc = kv.reserve(ctx, {{ctx, pos, pos + n_steps}});
    if (rc) return rc;
    int done = 0;
    rc = run_device_loop(ctx, G_ARGMAX_LOOP, token, pos, n_steps, forced, stop_on_bos, &done);
    if (rc) return rc;
    for (int i = 0; i < done; ++i) out_next[i] = ctx->h_gen[i];
    *n_done = done;
    return L2B_OK;
}

// Prompt prefill (SURVEY 8f.2; src/main.zig:996-1000 feeds prompt tokens through transformer() one
// at a time and throws their logits away).  All positions run back to back on the device with
// the next token forced, the classifier (60 % of stories15M's bytes) is skipped for every position
// whose logits nobody reads, and no position pays a host round trip.  On bandwidth-bound shapes
// (llama2-7B on one GPU) PF_MAXB = 4 positions additionally share each pass over the weights
// (prefill_gemm_kernel).  Per (row, position) the arithmetic is the decode step's own.
int32_t l2b_prefill(l2b_ctx *ctx, const int32_t *tokens, int32_t n_tokens, int32_t pos0, float *host_logits) {
    if (!ctx || !tokens || n_tokens <= 0) return fail(ctx, L2B_ERR_INVALID_ARG, "bad prefill arguments");
    int rc = check_step_args(ctx, tokens[0], pos0);
    if (rc) return rc;
    if (pos0 + n_tokens > ctx->cfg.seq_len) return fail(ctx, L2B_ERR_INVALID_ARG, "prompt runs past seq_len");
    for (int i = 0; i < n_tokens; ++i)
        if (tokens[i] < 0 || tokens[i] >= ctx->cfg.vocab_size) return fail(ctx, L2B_ERR_INVALID_ARG, "token out of range");
    const int n_silent = host_logits ? n_tokens - 1 : n_tokens;   // positions whose logits are dropped
    KvCall kv;
    rc = kv.reserve(ctx, {{ctx, pos0, pos0 + n_tokens}});
    if (rc) return rc;
    rc = pf_prepare(ctx);
    if (rc) return rc;
    if (n_silent > 0 && ctx->pf_ok) {
        // bandwidth-bound shapes: PF_MAXB positions share each pass over the weights
        rc = prefill_batched(ctx, tokens, n_silent, pos0);
        if (rc) return rc;
    } else if (n_silent > 0) {
        std::vector<int32_t> forced(n_silent);
        for (int i = 0; i < n_silent; ++i) forced[i] = tokens[i + 1 < n_tokens ? i + 1 : i];
        int done = 0;
        rc = run_device_loop(ctx, G_PREFILL_LOOP, tokens[0], pos0, n_silent, forced.data(), 0, &done);
        if (rc) return rc;
        if (done != n_silent) return fail(ctx, L2B_ERR_STATE, "prefill stopped early");
    }
    if (host_logits) return l2b_forward(ctx, tokens[n_tokens - 1], pos0 + n_tokens - 1, host_logits);
    return L2B_OK;
}

// Teacher forcing: tokens[i] at pos0 + i for i < n_tokens - 1, each position's log-probability of
// tokens[i + 1] and its greedy token.  Where l2b_prefill batches, the same groups of PF_MAXB positions
// as l2b_prefill(tokens, n_tokens - 1, pos0) with the argmax classifier and logprob_batch_kernel after
// each; otherwise the device loop G_SCORE_LOOP (a decode step with the argmax classifier,
// logprob_kernel, advance_kernel on the forced tokens tokens[1..]).
int32_t l2b_score(l2b_ctx *ctx, const int32_t *tokens, int32_t n_tokens, int32_t pos0, float *logprob,
                  int32_t *greedy) {
    if (!ctx) { g_create_error = "ctx is NULL"; return L2B_ERR_INVALID_ARG; }
    if (!tokens || !logprob || n_tokens < 1) return fail(ctx, L2B_ERR_INVALID_ARG, "bad score arguments");
    for (int i = 0; i < n_tokens; ++i)
        if (tokens[i] < 0 || tokens[i] >= ctx->cfg.vocab_size) return fail(ctx, L2B_ERR_INVALID_ARG, "token out of range");
    if (pos0 < 0 || (int64_t)pos0 + n_tokens - 1 > ctx->cfg.seq_len) return fail(ctx, L2B_ERR_INVALID_ARG, "score runs past seq_len");
    if (pos0 > ctx->n_appended) return fail(ctx, L2B_ERR_STATE, "pos0 skips ahead of the KV cache");
    if (ctx->world > 1)
        return fail(ctx, L2B_ERR_UNSUPPORTED, "l2b_score needs a single-GPU context (under tensor parallelism each rank holds only a slice of the vocabulary)");
    ctx->last_ms = 0.0f;
    ctx->last_launches = 0;
    const int n = n_tokens - 1;                               // positions scored
    if (n == 0) return L2B_OK;
    KvCall kv;
    int rc = kv.reserve(ctx, {{ctx, pos0, pos0 + n}});
    if (rc) return rc;
    rc = pf_prepare(ctx);
    if (rc) return rc;
    if (ctx->pf_ok) {
        rc = prefill_batched(ctx, tokens, n, pos0, true);
        if (rc) return rc;
    } else {
        int done = 0;
        rc = run_device_loop(ctx, G_SCORE_LOOP, tokens[0], pos0, n, tokens + 1, 0, &done);
        if (rc) return rc;
        if (done != n) return fail(ctx, L2B_ERR_STATE, "score stopped early");
    }
    L2B_CUDA(ctx, cudaMemcpy(logprob, ctx->score_lp, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
    if (greedy) L2B_CUDA(ctx, cudaMemcpy(greedy, ctx->score_greedy, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
    return L2B_OK;
}

}  // extern "C"

// The batch and ragged calls of one mode share their body: ragged == false is the batched step (one
// token per session, n_tok ignored).
static int forward_runs(l2b_ctx *const *sessions, int32_t n, bool ragged, const int32_t *n_tok, const int32_t *tokens,
                        const int32_t *pos, float *const *host_logits) {
    int rc = check_batch_args(sessions, n, tokens, pos, ragged, n_tok);
    if (rc) return rc;
    if (!host_logits) return fail(sessions[0], L2B_ERR_INVALID_ARG, "host_logits is NULL");
    for (int i = 0; i < n; ++i)
        if (!host_logits[i]) return fail(sessions[0], L2B_ERR_INVALID_ARG, "a host_logits entry is NULL");
    rc = step_sessions(sessions, n, ragged ? n_tok : nullptr, tokens, pos, MODE_LOGITS);
    if (rc) return rc;
    for (int i = 0; i < n; ++i)
        if (host_logits[i] != sessions[i]->h_logits)
            memcpy(host_logits[i], sessions[i]->h_logits, (size_t)sessions[i]->cfg.vocab_size * sizeof(float));
    return L2B_OK;
}

static int forward_argmax_runs(l2b_ctx *const *sessions, int32_t n, bool ragged, const int32_t *n_tok,
                               const int32_t *tokens, const int32_t *pos, int32_t *next) {
    int rc = check_batch_args(sessions, n, tokens, pos, ragged, n_tok);
    if (rc) return rc;
    if (!next) return fail(sessions[0], L2B_ERR_INVALID_ARG, "next is NULL");
    rc = step_sessions(sessions, n, ragged ? n_tok : nullptr, tokens, pos, MODE_ARGMAX);
    if (rc) return rc;
    for (int i = 0; i < n; ++i) next[i] = sessions[i]->h_ints[0];
    return L2B_OK;
}

// The sampler arguments of the batch, ragged and verify sample calls, checked before anything runs; on
// success filter_p[i] is session i's top-p as the kernels take it (< 0: no filter).
static int check_sample_args(l2b_ctx *s0, int32_t n, const float *temperature, const float *top_p,
                             const l2b_prob_index *cand, int32_t cand_cap, const int32_t *n_cand,
                             std::vector<float> &filter_p) {
    if (!temperature || !top_p) return fail(s0, L2B_ERR_INVALID_ARG, "temperature or top_p is NULL");
    if (s0->cfg.vocab_size < 2) return fail(s0, L2B_ERR_INVALID_ARG, "sampling needs vocab_size >= 2");
    filter_p.assign(n, -1.0f);
    for (int i = 0; i < n; ++i) {
        if (!(temperature[i] > 0.0f)) return fail(s0, L2B_ERR_INVALID_ARG, "temperature must be > 0 (use l2b_forward_argmax_batch for 0)");
        if (!(top_p[i] >= 0.0f && top_p[i] <= 1.0f)) return fail(s0, L2B_ERR_INVALID_ARG, "top_p must be in [0, 1]");
        const bool filter = (top_p[i] != 0.0f && top_p[i] != 1.0f);   // :1009
        if (filter && (!cand || !n_cand || cand_cap <= 0)) return fail(s0, L2B_ERR_INVALID_ARG, "candidate buffer missing");
        filter_p[i] = filter ? top_p[i] : -1.0f;
    }
    return L2B_OK;
}

static int forward_sample_runs(l2b_ctx *const *sessions, int32_t n, bool ragged, const int32_t *n_tok,
                               const int32_t *tokens, const int32_t *pos, const float *temperature,
                               const float *top_p, float *const *host_probs, l2b_prob_index *cand,
                               int32_t cand_cap, int32_t *n_cand) {
    int rc = check_batch_args(sessions, n, tokens, pos, ragged, n_tok);
    if (rc) return rc;
    std::vector<float> filter_p;
    rc = check_sample_args(sessions[0], n, temperature, top_p, cand, cand_cap, n_cand, filter_p);
    if (rc) return rc;
    rc = step_sessions(sessions, n, ragged ? n_tok : nullptr, tokens, pos, MODE_SAMPLE, temperature, filter_p.data());
    if (rc) return rc;
    for (int i = 0; i < n; ++i)
        copy_step_sample_out(sessions[i], filter_p[i] >= 0.0f, host_probs ? host_probs[i] : nullptr,
                        cand && cand_cap > 0 ? cand + (size_t)i * cand_cap : nullptr, cand_cap,
                        n_cand ? n_cand + i : nullptr);
    return L2B_OK;
}

extern "C" {

int32_t l2b_forward_batch(l2b_ctx *const *sessions, int32_t n, const int32_t *tokens, const int32_t *pos,
                          float *const *host_logits) {
    return forward_runs(sessions, n, false, nullptr, tokens, pos, host_logits);
}

int32_t l2b_forward_argmax_batch(l2b_ctx *const *sessions, int32_t n, const int32_t *tokens, const int32_t *pos,
                                 int32_t *next) {
    return forward_argmax_runs(sessions, n, false, nullptr, tokens, pos, next);
}

int32_t l2b_forward_sample_batch(l2b_ctx *const *sessions, int32_t n, const int32_t *tokens, const int32_t *pos,
                                 const float *temperature, const float *top_p, float *const *host_probs,
                                 l2b_prob_index *cand, int32_t cand_cap, int32_t *n_cand) {
    return forward_sample_runs(sessions, n, false, nullptr, tokens, pos, temperature, top_p, host_probs, cand,
                               cand_cap, n_cand);
}

int32_t l2b_forward_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens, const int32_t *tokens,
                           const int32_t *pos0, float *const *host_logits) {
    return forward_runs(sessions, n, true, n_tokens, tokens, pos0, host_logits);
}

int32_t l2b_forward_argmax_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens,
                                  const int32_t *tokens, const int32_t *pos0, int32_t *next) {
    return forward_argmax_runs(sessions, n, true, n_tokens, tokens, pos0, next);
}

int32_t l2b_forward_sample_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens,
                                  const int32_t *tokens, const int32_t *pos0, const float *temperature,
                                  const float *top_p, float *const *host_probs, l2b_prob_index *cand,
                                  int32_t cand_cap, int32_t *n_cand) {
    return forward_sample_runs(sessions, n, true, n_tokens, tokens, pos0, temperature, top_p, host_probs, cand,
                               cand_cap, n_cand);
}

// l2b_generate_argmax_batch where the batched step runs (pf_ok on s[0]): every step of every group of
// PF_MAXB sessions is enqueued up front on s[0]'s stream, with no host synchronise until the end.  The
// positions are launch arguments (pos[i] + step, held at seq_len - 1 once session i is past its limit);
// the tokens stay on the device: batch_advance_kernel writes each session's next token into the call's
// token array, which the next step's qkv kernel embeds.  A stopped session's vector still flows through
// its group, appends no KV row (the done flags are qkv's skip mask) and its outputs are ignored; once
// every session has stopped (CTL_DONE on s[0]) the launches still queued return at once.
static int generate_batched(l2b_ctx *const *s, int n, const int32_t *tokens, const int32_t *pos, int n_steps,
                            const int32_t *forced, const int *limit, int stop_on_bos, int32_t *out_next,
                            int32_t *n_done) {
    l2b_ctx *ctx = s[0];
    const int S = ctx->cfg.seq_len;
    int stride = 0;                          // steps of the longest-running session
    for (int i = 0; i < n; ++i) stride = limit[i] > stride ? limit[i] : stride;
    // the call's device ints: tokens, done flags, limits [n] each, the live count, forced [n][stride], then
    // the results: n_done [n] and out_next [n][stride]
    const size_t o_tok = 0, o_done = (size_t)n, o_lim = 2 * (size_t)n, o_live = 3 * (size_t)n;
    const size_t o_forced = o_live + 1, o_ndone = o_forced + (size_t)n * stride, o_out = o_ndone + n;
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<int> h(o_out + (size_t)n * stride, -1);
    for (int i = 0; i < n; ++i) {
        h[o_tok + i] = tokens[i];
        h[o_done + i] = 0;
        h[o_ndone + i] = 0;
        h[o_lim + i] = limit[i];
        if (forced)
            for (int k = 0; k < limit[i]; ++k) h[o_forced + (size_t)i * stride + k] = forced[(size_t)i * n_steps + k];
    }
    h[o_live] = n;
    int rc = batched_begin(ctx, h.data(), h.size(), tokens[0], pos[0]);
    if (rc) return rc;
    int *d = ctx->call_ints;
    BatchAdvanceParams a{};
    a.ctl = ctx->ctl;
    a.amax = ctx->pf_amax;
    a.forced = forced ? d + o_forced : nullptr;
    a.limit = d + o_lim;
    a.tokens = d + o_tok; a.done = d + o_done; a.n_done = d + o_ndone; a.out_next = d + o_out;
    a.live = d + o_live;
    a.stride = stride;
    a.stop_on_bos = stop_on_bos ? 1 : 0;
    for (int step = 0; step < stride; ++step) {
        for (int g = 0; g < n; g += PF_MAXB) {
            const int nb = n - g < PF_MAXB ? n - g : PF_MAXB;
            int p[PF_MAXB];
            for (int b = 0; b < nb; ++b) p[b] = pos[g + b] + step < S ? pos[g + b] + step : S - 1;
            rc = batched_layers(ctx, s + g, p, nb, d + o_tok + g, d + o_done + g);
            if (rc) return rc;
            rc = batched_classifier(ctx, nb, true);
            if (rc) return rc;
            a.g0 = g; a.nb = nb; a.step = step;
            void *args[] = {&a};
            rc = launch_small(ctx, (const void *)batch_advance_kernel, dim3(1), dim3(PF_MAXB), args, ctx->stream, true);
            if (rc) return rc;
        }
    }
    std::vector<int> back(h.size() - o_ndone);     // n_done [n], then out_next [n][stride]
    rc = batched_end(ctx, back.data(), o_ndone, back.size());
    if (rc) return rc;
    for (int i = 0; i < n; ++i) {
        n_done[i] = back[i];
        for (int k = 0; k < n_done[i]; ++k) out_next[(size_t)i * n_steps + k] = back[n + (size_t)i * stride + k];
        if (pos[i] + n_done[i] > s[i]->n_appended) s[i]->n_appended = pos[i] + n_done[i];
    }
    return L2B_OK;
}

// l2b_generate_argmax_batch elsewhere: each session's own device loop (l2b_generate_argmax's graph
// replays) on its own stream, the sessions' replays interleaved step by step, one synchronise for all
static int generate_each(l2b_ctx *const *s, int n, const int32_t *tokens, const int32_t *pos, int n_steps,
                         const int32_t *forced, const int *limit, int stop_on_bos, int32_t *out_next,
                         int32_t *n_done) {
    std::vector<DeviceLoop> loops;
    for (int i = 0; i < n; ++i)
        loops.push_back(DeviceLoop{s[i], tokens[i], pos[i], limit[i], forced ? forced + (size_t)i * n_steps : nullptr, true});
    int rc = enqueue_device_loops(loops, G_ARGMAX_LOOP, stop_on_bos);
    if (rc) return rc;
    rc = finish_device_loops(loops);
    if (rc) return rc;
    int launches = 0;
    for (int i = 0; i < n; ++i) {
        launches += loops[i].launches;
        n_done[i] = loops[i].done;
        for (int k = 0; k < n_done[i]; ++k) out_next[(size_t)i * n_steps + k] = s[i]->h_gen[k];
    }
    s[0]->last_launches = launches;
    return L2B_OK;
}

int32_t l2b_generate_argmax_batch(l2b_ctx *const *sessions, int32_t n, const int32_t *tokens, const int32_t *pos,
                                  int32_t n_steps, const int32_t *forced, int32_t stop_on_bos, int32_t *out_next,
                                  int32_t *n_done) {
    int rc = check_batch_args(sessions, n, tokens, pos);
    if (rc) return rc;
    l2b_ctx *s0 = sessions[0];
    if (!out_next || !n_done || n_steps < 0) return fail(s0, L2B_ERR_INVALID_ARG, "bad generate arguments");
    std::vector<int> limit(n);
    for (int i = 0; i < n; ++i) {
        const int left = s0->cfg.seq_len - pos[i];
        limit[i] = n_steps < left ? n_steps : left;                   // :992-993, per session
        rc = check_forced(s0, forced ? forced + (size_t)i * n_steps : nullptr, limit[i]);
        if (rc) return rc;
    }
    for (int i = 0; i < n; ++i) n_done[i] = 0;
    if (n_steps == 0) return L2B_OK;
    std::vector<KvRange> ranges;
    for (int i = 0; i < n; ++i) ranges.push_back(KvRange{sessions[i], pos[i], pos[i] + limit[i]});
    KvCall kv;
    rc = kv.reserve(s0, ranges);
    if (rc) return rc;
    rc = pf_prepare(s0);
    if (rc) return rc;
    if (s0->pf_ok) return generate_batched(sessions, n, tokens, pos, n_steps, forced, limit.data(), stop_on_bos, out_next, n_done);
    return generate_each(sessions, n, tokens, pos, n_steps, forced, limit.data(), stop_on_bos, out_next, n_done);
}

// l2b_verify_argmax_ragged where the batched step runs (pf_ok on s[0]): the runs' vectors, back to back, go
// PF_MAXB per pass over the weights as in step_sessions, each on its own session's cache at its own
// position, and after each group's argmax classifier verify_accept_kernel decides the runs it holds.  Every
// group is enqueued up front; once every run is decided (CTL_DONE on s[0]) the groups still queued return
// at once.  The call's device ints: tokens [total], greedy [total], n_accept [n] (-1: undecided) and the
// undecided count.
static int verify_batched(l2b_ctx *const *s, int n, const int32_t *n_tok, const int32_t *tokens, const int32_t *pos,
                          int stop_on_bos, int32_t *greedy, int32_t *n_accept) {
    l2b_ctx *ctx = s[0];
    const RunVectors r = expand_runs(s, n, n_tok, pos);   // vector v runs tokens[v]
    const int total = (int)r.kv.size();
    const size_t o_tok = 0, o_greedy = (size_t)total, o_acc = 2 * (size_t)total, o_live = o_acc + n, size = o_live + 1;
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<int> h(size, -1);
    for (int v = 0; v < total; ++v) h[o_tok + v] = tokens[v];
    h[o_live] = n;
    int rc = batched_begin(ctx, h.data(), size, tokens[0], pos[0]);
    if (rc) return rc;
    int *d = ctx->call_ints;
    VerifyAcceptParams a{};
    a.ctl = ctx->ctl;
    a.amax = ctx->pf_amax;
    a.tokens = d + o_tok; a.greedy = d + o_greedy; a.n_accept = d + o_acc; a.live = d + o_live;
    a.stop_on_bos = stop_on_bos ? 1 : 0;
    for (int g = 0; g < total; g += PF_MAXB) {
        const int nb = total - g < PF_MAXB ? total - g : PF_MAXB;
        rc = batched_layers(ctx, r.kv.data() + g, r.pos.data() + g, nb, d + o_tok + g, nullptr);
        if (rc) return rc;
        rc = batched_classifier(ctx, nb, true);
        if (rc) return rc;
        a.g0 = g;
        a.nb = nb;
        for (int b = 0; b < nb; ++b) {
            a.run[b] = r.run[g + b];
            a.j[b] = r.j[g + b];
            a.last[b] = n_tok[r.run[g + b]] - 1;
        }
        void *args[] = {&a};
        rc = launch_small(ctx, (const void *)verify_accept_kernel, dim3(1), dim3(32), args, ctx->stream, true);
        if (rc) return rc;
    }
    std::vector<int> back((size_t)total + n);     // greedy [total], then n_accept [n]
    rc = batched_end(ctx, back.data(), o_greedy, back.size());
    if (rc) return rc;
    for (int i = 0, off = 0; i < n; off += n_tok[i], ++i) {
        const int acc = back[(size_t)total + i];
        if (acc < 0) return fail(ctx, L2B_ERR_STATE, "verify: a run was left undecided");
        n_accept[i] = acc;
        for (int j = 0; j <= acc; ++j) greedy[off + j] = back[off + j];
    }
    return L2B_OK;
}

// l2b_verify_argmax_ragged elsewhere: each run is l2b_score's device loop (G_SCORE_LOOP: the decode step
// with the argmax classifier) on its own session and stream, forced through the run's drafts and, after
// its last position, a placeholder that nothing reads as a token; the sessions' replays are interleaved,
// one synchronise for all.  Every position runs; the acceptance is decided on the host from score_greedy.
static int verify_each(l2b_ctx *const *s, int n, const int32_t *n_tok, const int32_t *tokens, const int32_t *pos,
                       int stop_on_bos, int32_t *greedy, int32_t *n_accept) {
    std::vector<std::vector<int32_t>> forced(n);
    std::vector<DeviceLoop> loops;
    for (int i = 0, off = 0; i < n; off += n_tok[i], ++i) {
        forced[i].assign(tokens + off + 1, tokens + off + n_tok[i]);
        forced[i].push_back(tokens[off]);
        loops.push_back(DeviceLoop{s[i], tokens[off], pos[i], n_tok[i], forced[i].data(), true});
    }
    int rc = enqueue_device_loops(loops, G_SCORE_LOOP, 0);
    if (rc) return rc;
    rc = finish_device_loops(loops);
    if (rc) return rc;
    int launches = 0;
    std::vector<int32_t> gr;
    for (int i = 0, off = 0; i < n; off += n_tok[i], ++i) {
        l2b_ctx *c = s[i];
        launches += loops[i].launches;
        if (loops[i].done != n_tok[i]) return fail(s[0], L2B_ERR_STATE, "verify stopped early");
        gr.resize(n_tok[i]);
        L2B_CUDA(s[0], cudaSetDevice(c->device));
        L2B_CUDA(s[0], cudaMemcpy(gr.data(), c->score_greedy, gr.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
        int acc = 0;
        while (acc < n_tok[i] - 1 && !(stop_on_bos && gr[acc] == 1) && tokens[off + acc + 1] == gr[acc]) ++acc;
        n_accept[i] = acc;
        for (int j = 0; j <= acc; ++j) greedy[off + j] = gr[j];
    }
    s[0]->last_launches = launches;
    return L2B_OK;
}

int32_t l2b_verify_argmax_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens, const int32_t *tokens,
                                 const int32_t *pos0, int32_t stop_on_bos, int32_t *greedy, int32_t *n_accept) {
    int rc = check_batch_args(sessions, n, tokens, pos0, true, n_tokens);
    if (rc) return rc;
    l2b_ctx *s0 = sessions[0];
    if (!greedy || !n_accept) return fail(s0, L2B_ERR_INVALID_ARG, "greedy or n_accept is NULL");
    if (s0->world > 1) return fail(s0, L2B_ERR_UNSUPPORTED, "l2b_verify_argmax_ragged needs a single-GPU model");
    std::vector<KvRange> ranges;
    for (int i = 0; i < n; ++i) ranges.push_back(KvRange{sessions[i], pos0[i], pos0[i] + n_tokens[i]});
    KvCall kv;
    rc = kv.reserve(s0, ranges);
    if (rc) return rc;
    rc = pf_prepare(s0);
    if (rc) return rc;
    rc = s0->pf_ok ? verify_batched(sessions, n, n_tokens, tokens, pos0, stop_on_bos, greedy, n_accept)
                   : verify_each(sessions, n, n_tokens, tokens, pos0, stop_on_bos, greedy, n_accept);
    if (rc) return rc;
    for (int i = 0; i < n; ++i) sessions[i]->n_appended = pos0[i] + n_accept[i] + 1;
    return L2B_OK;
}

// Greedy speculative decoding: rounds of (the draft's device loop proposes kk tokens, one verify of
// [token, d_1 .. d_kk] on the target).  dp counts the stream positions the draft holds rows for: after a
// round that accepted a < kk drafts the draft's rows up to p + a hold the stream, after one that accepted
// all it never ran d_kk, and after a round without proposals it did not run at all.  The next draft loop
// starts at dp and is forced through the stream up to the target's token (the catch-up), then runs free.
int32_t l2b_generate_speculative(l2b_ctx *target, l2b_ctx *draft, int32_t token, int32_t pos, int32_t n_steps,
                                 int32_t k, int32_t stop_on_bos, int32_t *out_next, int32_t *n_done,
                                 int32_t *n_rounds) {
    if (!target) { g_create_error = "target is NULL"; return L2B_ERR_INVALID_ARG; }
    if (!draft || !out_next || !n_done) return fail(target, L2B_ERR_INVALID_ARG, "draft, out_next or n_done is NULL");
    if (draft == target) return fail(target, L2B_ERR_INVALID_ARG, "the draft is the target");
    if (k < 0 || k > L2B_SPECULATIVE_MAX_K) return fail(target, L2B_ERR_INVALID_ARG, "k outside [0, L2B_SPECULATIVE_MAX_K]");
    if (n_steps < 0) return fail(target, L2B_ERR_INVALID_ARG, "n_steps < 0");
    const int S = target->cfg.seq_len;
    if (token < 0 || token >= target->cfg.vocab_size) return fail(target, L2B_ERR_INVALID_ARG, "token out of range");
    if (pos < 0 || pos >= S) return fail(target, L2B_ERR_INVALID_ARG, "pos out of range");
    if (draft->cfg.vocab_size != target->cfg.vocab_size) return fail(target, L2B_ERR_INVALID_ARG, "the draft has another vocabulary size");
    if (draft->cfg.seq_len < S) return fail(target, L2B_ERR_INVALID_ARG, "the draft's seq_len is below the target's");
    if (target->world > 1 || draft->world > 1)
        return fail(target, L2B_ERR_UNSUPPORTED, "l2b_generate_speculative needs single-GPU target and draft");
    if (pos > target->n_appended || pos > draft->n_appended)
        return fail(target, L2B_ERR_STATE, "pos skips ahead of the target's or the draft's KV cache");
    if (n_steps > S - pos) n_steps = S - pos;                 // :992-993
    // every row either model may write, up front, so a refused call changes neither; the rounds' own calls
    // then only re-take pages they released in between
    KvCall kv;
    std::vector<KvRange> ranges{{target, pos, pos + n_steps}};
    if (draft->paged) ranges.push_back(KvRange{draft, pos, pos + n_steps});
    if (!target->paged && draft->paged) ranges.erase(ranges.begin());
    if (int rc = kv.reserve(target, ranges)) return rc;
    float ms = 0.0f;
    int launches = 0, rounds = 0, done = 0;
    std::vector<int32_t> hist(1, token);   // hist[q - pos]: the stream's token at position q
    std::vector<int32_t> run, forced, out(S), gr(L2B_SPECULATIVE_MAX_K + 1);
    int p = pos, dp = pos;                 // the target's next position; the stream positions the draft holds
    bool stopped = false;
    while (done < n_steps && !stopped) {
        int kk = k < n_steps - done - 1 ? k : n_steps - done - 1;
        if (kk > S - 1 - p) kk = S - 1 - p;
        run.assign(1, hist[p - pos]);
        if (kk > 0) {
            const int lag = p - dp;        // forced through the stream tokens at dp + 1 .. p, then free
            forced.assign(hist.begin() + (dp - pos) + 1, hist.end());
            forced.resize((size_t)lag + kk, -1);
            int nd = 0;
            int rc = l2b_generate_argmax(draft, hist[dp - pos], dp, lag + kk, forced.data(), 0, out.data(), &nd);
            if (rc) return fail(target, rc, draft->err.c_str());
            if (nd != lag + kk) return fail(target, L2B_ERR_STATE, "the draft loop stopped early");
            ms += draft->last_ms;
            launches += draft->last_launches;
            run.insert(run.end(), out.begin() + lag, out.begin() + lag + kk);
        }
        const int32_t nt = kk + 1;
        int32_t acc = 0;
        int rc = l2b_verify_argmax_ragged(&target, 1, &nt, run.data(), &p, stop_on_bos, gr.data(), &acc);
        if (rc) return rc;
        ms += target->last_ms;
        launches += target->last_launches;
        ++rounds;
        const int emit = acc + 1 < n_steps - done ? acc + 1 : n_steps - done;
        for (int j = 0; j < emit; ++j) {
            out_next[done + j] = gr[j];
            hist.push_back(gr[j]);
        }
        if (kk > 0) dp = p + (acc + 1 < kk ? acc + 1 : kk);
        done += emit;
        p += emit;
        stopped = stop_on_bos && gr[emit - 1] == 1;
    }
    const int end = pos + done;
    if (dp < end) {                        // the draft's missing rows of the stream: one prefill
        const int rc = l2b_prefill(draft, hist.data() + (dp - pos), end - dp, dp, nullptr);
        if (rc) return fail(target, rc, draft->err.c_str());
        ms += draft->last_ms;
        launches += draft->last_launches;
    }
    target->n_appended = end;
    draft->n_appended = end;
    target->last_ms = ms;
    target->last_launches = launches;
    *n_done = done;
    if (n_rounds) *n_rounds = rounds;
    return L2B_OK;
}

// l2b_verify_sample_ragged where the batched step runs (pf_ok on s[0]): the runs' vectors go PF_MAXB per pass
// as in step_sessions, and every vector is an output: each pass runs the classifier and sample_prep_batch_kernel
// over all its rows, row v's candidates to call_cand + v * kCandCap and its count to the call's ints.  The
// probabilities of each pass (when wanted) and, at the end, every position's candidates (when some session
// filters) go to the pinned staging h_call in one copy each; the counts come back through batched_end.  The
// call's device ints: tokens [total], then counts [total].
static int verify_sample_batched(l2b_ctx *const *s, int n, const int32_t *n_tok, const int32_t *tokens, const int32_t *pos,
                                 const float *temperature, const float *filter_p, float *host_probs,
                                 l2b_prob_index *cand, int32_t cand_cap, int32_t *n_cand) {
    l2b_ctx *ctx = s[0];
    const RunVectors r = expand_runs(s, n, n_tok, pos);   // vector v runs tokens[v]
    const int total = (int)r.kv.size(), V = ctx->cfg.vocab_size;
    bool want_cand = false;
    for (int i = 0; i < n; ++i) want_cand |= filter_p[i] >= 0.0f;
    const size_t probs_bytes = host_probs ? (size_t)total * V * sizeof(float) : 0;
    const size_t bytes = probs_bytes + (want_cand ? (size_t)total * kCandCap * sizeof(ProbIndex) : 0);
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    if (ctx->h_call_bytes < bytes) {
        if (ctx->h_call) L2B_CUDA(ctx, cudaFreeHost(ctx->h_call));
        ctx->h_call = nullptr;
        ctx->h_call_bytes = 0;
        if (cudaHostAlloc((void **)&ctx->h_call, bytes, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            ctx->h_call = nullptr;
            return fail(ctx, L2B_ERR_OOM, "cudaHostAlloc of the verify staging failed");
        }
        ctx->h_call_bytes = bytes;
    }
    float *h_probs = reinterpret_cast<float *>(ctx->h_call);
    ProbIndex *h_cand = reinterpret_cast<ProbIndex *>(ctx->h_call + probs_bytes);
    int rc = want_cand ? call_buf_reserve(ctx, ctx->call_cand, ctx->call_cand_cap, (size_t)total * kCandCap) : L2B_OK;
    if (rc) return rc;
    std::vector<int> h(2 * (size_t)total, 0);
    std::copy(tokens, tokens + total, h.begin());
    rc = batched_begin(ctx, h.data(), h.size(), tokens[0], pos[0]);
    if (rc) return rc;
    int *d = ctx->call_ints;
    cudaStream_t st = ctx->stream;
    for (int g = 0; g < total; g += PF_MAXB) {
        const int nb = total - g < PF_MAXB ? total - g : PF_MAXB;
        rc = batched_layers(ctx, r.kv.data() + g, r.pos.data() + g, nb, d + g, nullptr);
        if (rc) return rc;
        rc = batched_classifier(ctx, nb, false);
        if (rc) return rc;
        float lt[PF_MAXB], lp[PF_MAXB];
        ProbIndex *lc[PF_MAXB];
        int *ln[PF_MAXB];
        for (int b = 0; b < nb; ++b) {
            const int v = g + b, i = r.run[v];
            lt[b] = temperature[i];
            lp[b] = filter_p[i];
            lc[b] = want_cand ? ctx->call_cand + (size_t)v * kCandCap : nullptr;   // not read without the filter
            ln[b] = d + total + v;
        }
        rc = launch_sample_prep_batch(ctx, nb, lt, lp, lc, ln);
        if (rc) return rc;
        if (host_probs)
            L2B_CUDA(ctx, cudaMemcpyAsync(h_probs + (size_t)g * V, ctx->pf_logits, (size_t)nb * V * sizeof(float),
                                          cudaMemcpyDeviceToHost, st));
    }
    if (want_cand)
        L2B_CUDA(ctx, cudaMemcpyAsync(h_cand, ctx->call_cand, (size_t)total * kCandCap * sizeof(ProbIndex),
                                      cudaMemcpyDeviceToHost, st));
    std::vector<int> counts(total);
    rc = batched_end(ctx, counts.data(), total, total);
    if (rc) return rc;
    for (int v = 0; v < total; ++v)
        copy_sample_out(V, h_probs + (size_t)v * V, h_cand + (size_t)v * kCandCap, counts[v], filter_p[r.run[v]] >= 0.0f,
                        host_probs ? host_probs + (size_t)v * V : nullptr,
                        cand && cand_cap > 0 ? cand + (size_t)v * cand_cap : nullptr, cand_cap, n_cand ? n_cand + v : nullptr);
    for (int i = 0; i < n; ++i)
        if (pos[i] + n_tok[i] > s[i]->n_appended) s[i]->n_appended = pos[i] + n_tok[i];
    return L2B_OK;
}

// l2b_verify_sample_ragged elsewhere: every position is l2b_forward_sample's own step (G_SAMPLE) on its
// session, and its output is copied out as that call copies it.  Each step ends in a synchronise: ev0 .. ev1
// spans them all.
static int verify_sample_each(l2b_ctx *const *s, int n, const int32_t *n_tok, const int32_t *tokens, const int32_t *pos,
                              const float *temperature, const float *filter_p, float *host_probs,
                              l2b_prob_index *cand, int32_t cand_cap, int32_t *n_cand) {
    l2b_ctx *ctx = s[0];
    const int V = ctx->cfg.vocab_size;
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    int launches = 0;
    for (int i = 0, v = 0; i < n; ++i)
        for (int j = 0; j < n_tok[i]; ++j, ++v) {
            int rc = run_step(s[i], tokens[v], pos[i] + j, G_SAMPLE, temperature[i], filter_p[i]);
            if (rc) { ctx->err = s[i]->err; return rc; }
            launches += s[i]->last_launches;
            copy_step_sample_out(s[i], filter_p[i] >= 0.0f, host_probs ? host_probs + (size_t)v * V : nullptr,
                                 cand && cand_cap > 0 ? cand + (size_t)v * cand_cap : nullptr, cand_cap,
                                 n_cand ? n_cand + v : nullptr);
        }
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev1, s[n - 1]->stream));
    L2B_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
    L2B_CUDA(ctx, cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
    ctx->last_launches = launches;
    return L2B_OK;
}

int32_t l2b_verify_sample_ragged(l2b_ctx *const *sessions, int32_t n, const int32_t *n_tokens, const int32_t *tokens,
                                 const int32_t *pos0, const float *temperature, const float *top_p, float *host_probs,
                                 l2b_prob_index *cand, int32_t cand_cap, int32_t *n_cand) {
    int rc = check_batch_args(sessions, n, tokens, pos0, true, n_tokens);
    if (rc) return rc;
    l2b_ctx *s0 = sessions[0];
    std::vector<float> filter_p;
    rc = check_sample_args(s0, n, temperature, top_p, cand, cand_cap, n_cand, filter_p);
    if (rc) return rc;
    int64_t total = 0;
    for (int i = 0; i < n; ++i) total += n_tokens[i];
    const int64_t per_pos = 4ll * s0->cfg.vocab_size + (int64_t)kCandCap * sizeof(ProbIndex);
    const int64_t cap = std::max<int64_t>((int64_t)n * (L2B_SPECULATIVE_MAX_K + 1), L2B_VERIFY_SAMPLE_STAGE_BYTES / per_pos);
    if (total > cap) return fail(s0, L2B_ERR_INVALID_ARG, "more positions than the verify staging holds (see L2B_VERIFY_SAMPLE_STAGE_BYTES)");
    if (s0->world > 1) return fail(s0, L2B_ERR_UNSUPPORTED, "l2b_verify_sample_ragged needs a single-GPU model");
    std::vector<KvRange> ranges;
    for (int i = 0; i < n; ++i) ranges.push_back(KvRange{sessions[i], pos0[i], pos0[i] + n_tokens[i]});
    KvCall kv;
    rc = kv.reserve(s0, ranges);
    if (rc) return rc;
    rc = pf_prepare(s0);
    if (rc) return rc;
    return s0->pf_ok ? verify_sample_batched(sessions, n, n_tokens, tokens, pos0, temperature, filter_p.data(), host_probs,
                                             cand, cand_cap, n_cand)
                     : verify_sample_each(sessions, n, n_tokens, tokens, pos0, temperature, filter_p.data(), host_probs,
                                          cand, cand_cap, n_cand);
}

// ---- beam search (l2b_beam_search) ----------------------------------------------------------------------

// logprob_topk_batch_kernel on nb rows of vocab_size logits, vocab_size apart, on ctx's stream: k best of
// row b to out[b * k ..]
static int launch_logprob_topk(l2b_ctx *ctx, const float *logits, int nb, int k, ProbIndex *out) {
    LogprobTopkParams p{ctx->ctl, logits, ctx->cfg.vocab_size, ctx->cfg.vocab_size, k, out};
    void *args[] = {&p};
    return launch_small(ctx, (const void *)logprob_topk_batch_kernel, dim3(nb), dim3(LOGPROB_THREADS), args, ctx->stream, true);
}

// A hypothesis: its tokens after the start token, its cumulative log-probability c, when it was made (step,
// position in that step's pool) and, once finished, its own references to its parent's pages.
struct BeamHyp {
    std::vector<int> toks;
    float c = 0.0f;
    int step = -1, at = 0, slot = -1;        // slot: the beam session a live hypothesis is in
    std::vector<void *> pages;
};
static uint32_t beam_fkey(float v) {         // the order of argmax_key's high word: larger float, larger key
    uint32_t u;
    memcpy(&u, &v, sizeof u);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// the result order: larger normalised score fl(c / len) (length penalty 1), then larger c, then earlier
static bool beam_better(const BeamHyp &a, const BeamHyp &b) {
    const uint32_t na = beam_fkey(a.c / (float)a.toks.size()), nb = beam_fkey(b.c / (float)b.toks.size());
    if (na != nb) return na > nb;
    if (a.c != b.c) return beam_fkey(a.c) > beam_fkey(b.c);
    return a.step != b.step ? a.step < b.step : a.at < b.at;
}
// new references to session s's pages [0, np)
static std::vector<void *> beam_take(l2b_ctx *s, int np) {
    std::vector<void *> v(s->pages.begin(), s->pages.begin() + np);
    for (void *pg : v)
        if (pg) ++kv_pool(s)->refs[pg];
    return v;
}
static void beam_put(KvPool *pool, std::vector<void *> &v) {
    for (void *pg : v)
        if (pg) kv_page_put(pool, pg);
    v.clear();
}
// session s gives up its pages and holds v (whose references pass to it) with n positions appended
static void beam_assign(l2b_ctx *s, const std::vector<void *> &v, int n) {
    for (int j = 0; j < s->n_pages; ++j) kv_drop(s, j);
    for (size_t j = 0; j < v.size(); ++j) {
        s->pages[j] = v[j];
        kv_tab_set(s, (int)j, v[j]);
    }
    s->n_appended = n;
}

// The search of l2b_beam_search on validated arguments (n_steps > 0, a paged model).  The live hypotheses are
// in beams[0 .. live.size()), each holding its pages; the finished ones hold theirs in fin.  Batched: the live
// hypotheses go PF_MAXB per pass through batched_layers and batched_classifier on beams[0]'s stream and
// buffers, and logprob_topk_batch_kernel reads pf_logits.  Otherwise each runs run_step(G_LOGITS) and the
// kernel reads its logits.  Only live.size() * K (lp, index) pairs come back per step.
struct BeamSearch {
    l2b_ctx *src, *lead;
    l2b_ctx *const *beams;
    int B, K, pos, token;
    bool stop;
    std::vector<BeamHyp> live, fin;
    int launches = 0, ran = 0;

    int err_from(l2b_ctx *c, int rc) {
        if (c != src) src->err = c->err;
        return rc;
    }
    int upload_all() {
        for (int i = 0; i < B; ++i)
            if (int rc = kv_tab_upload(beams[i])) return err_from(beams[i], rc);
        return L2B_OK;
    }
    // runs the last token of every live hypothesis at pos + t; their candidates to lead->h_cand
    int step(int t) {
        const int nl = (int)live.size();
        std::vector<KvRange> r;
        for (int j = 0; j < nl; ++j) r.push_back(KvRange{beams[j], pos + t, pos + t + 1});
        int rc = kv_reserve(src, r);
        if (rc) return rc;
        std::vector<int> last(nl), at(nl, pos + t);
        for (int j = 0; j < nl; ++j) last[j] = live[j].toks.empty() ? token : live[j].toks.back();
        cudaStream_t st = lead->stream;
        L2B_CUDA(src, cudaSetDevice(lead->device));
        if (lead->pf_ok) {
            lead->last_launches = 0;
            L2B_CUDA(src, cudaMemcpyAsync(lead->call_ints, last.data(), nl * sizeof(int), cudaMemcpyHostToDevice, st));
            for (int g = 0; g < nl; g += PF_MAXB) {
                const int nb = std::min(PF_MAXB, nl - g);
                if ((rc = batched_layers(lead, beams + g, at.data() + g, nb, lead->call_ints + g, nullptr)) ||
                    (rc = batched_classifier(lead, nb, false)) ||
                    (rc = launch_logprob_topk(lead, lead->pf_logits, nb, K, lead->call_cand + (size_t)g * K)))
                    return err_from(lead, rc);
            }
            launches += lead->last_launches;
        } else {
            for (int j = 0; j < nl; ++j) {
                if ((rc = run_step(beams[j], last[j], pos + t, G_LOGITS, 1.0f, 0.0f))) return err_from(beams[j], rc);
                launches += beams[j]->last_launches;
            }
            lead->last_launches = 0;
            for (int j = 0; j < nl; ++j)
                if ((rc = launch_logprob_topk(lead, beams[j]->logits, 1, K, lead->call_cand + (size_t)j * K))) return err_from(lead, rc);
            launches += lead->last_launches;
        }
        L2B_CUDA(src, cudaMemcpyAsync(lead->h_cand, lead->call_cand, (size_t)nl * K * sizeof(ProbIndex), cudaMemcpyDeviceToHost, st));
        L2B_CUDA(src, cudaStreamSynchronize(st));
        L2B_CUDA(src, cudaGetLastError());
        for (int j = 0; j < nl; ++j) beams[j]->n_appended = pos + t + 1;
        return L2B_OK;
    }
    // the selection after step t, and the page remap: slot j takes its parent's pages [0, np)
    int select(int t) {
        struct Cand { float score; int h, r; };
        const int nl = (int)live.size(), np = (pos + t + 1 + KV_PAGE_ROWS - 1) / KV_PAGE_ROWS;
        const ProbIndex *hc = lead->h_cand;
        std::vector<Cand> cand;
        for (int h = 0; h < nl; ++h)
            for (int r = 0; r < K; ++r) cand.push_back(Cand{live[h].c + hc[h * K + r].prob, h, r});
        std::sort(cand.begin(), cand.end(), [](const Cand &a, const Cand &b) {
            const uint32_t ka = beam_fkey(a.score), kb = beam_fkey(b.score);
            return ka != kb ? ka > kb : a.h != b.h ? a.h < b.h : a.r < b.r;
        });
        std::vector<BeamHyp> next;
        std::vector<std::vector<void *>> lists;
        for (int q = 0; q < (int)cand.size() && (int)next.size() < B; ++q) {
            const Cand &x = cand[q];
            BeamHyp y;
            y.toks = live[x.h].toks;
            y.toks.push_back(hc[x.h * K + x.r].index);
            y.c = x.score;
            y.step = t;
            y.at = q;
            if (stop && y.toks.back() == 1) {   // BOS: finished when it ranks among the first B, else dropped
                if (q >= B) continue;
                y.pages = beam_take(beams[x.h], np);
                fin.push_back(std::move(y));
                std::stable_sort(fin.begin(), fin.end(), beam_better);
                if ((int)fin.size() > B) {
                    beam_put(kv_pool(src), fin.back().pages);
                    fin.pop_back();
                }
                continue;
            }
            y.slot = (int)next.size();
            lists.push_back(beam_take(beams[x.h], np));
            next.push_back(std::move(y));
        }
        for (int j = 0; j < B; ++j) beam_assign(beams[j], j < (int)lists.size() ? lists[j] : std::vector<void *>(), pos + t + 1);
        live = std::move(next);
        return upload_all();
    }
    int run(int n_steps) {
        const int np0 = (pos + KV_PAGE_ROWS - 1) / KV_PAGE_ROWS;
        for (int i = 0; i < B; ++i) beam_assign(beams[i], beam_take(src, np0), pos);
        int rc = upload_all();
        if (rc) return rc;
        live.assign(1, BeamHyp());
        const int T = std::min(n_steps, src->cfg.seq_len - pos);
        for (int t = 0; t < T; ++t) {
            if ((rc = step(t)) || (rc = select(t))) return rc;
            ran = t + 1;
            if (stop && (int)fin.size() == B) {
                const BeamHyp &w = fin.back();
                if (w.c / (float)w.toks.size() >= live[0].c / (float)(t + 1)) break;
            }
        }
        return L2B_OK;
    }
    // beams[i] take the best B of fin and live; every other reference goes back
    int finish(int n_steps, int32_t *out_tokens, int32_t *out_len, float *out_logprob) {
        std::vector<BeamHyp> all = std::move(fin);
        fin.clear();
        for (BeamHyp &h : live) all.push_back(std::move(h));
        std::stable_sort(all.begin(), all.end(), beam_better);
        const int np = (pos + ran + KV_PAGE_ROWS - 1) / KV_PAGE_ROWS;
        std::vector<std::vector<void *>> lists(B);
        for (int i = 0; i < B; ++i) {
            if (all[i].slot >= 0) lists[i] = beam_take(beams[all[i].slot], np);
            else lists[i].swap(all[i].pages);
        }
        for (BeamHyp &h : all) beam_put(kv_pool(src), h.pages);
        for (int i = 0; i < B; ++i) {
            const BeamHyp &h = all[i];
            beam_assign(beams[i], lists[i], pos + (int)h.toks.size());
            std::copy(h.toks.begin(), h.toks.end(), out_tokens + (size_t)i * n_steps);
            out_len[i] = (int)h.toks.size();
            out_logprob[i] = h.c;
        }
        return upload_all();
    }
    // after a failure: every beam holds nothing and has 0 positions appended; src was never written
    void abandon() {
        for (int i = 0; i < B; ++i) {
            beam_assign(beams[i], std::vector<void *>(), 0);
            kv_tab_upload(beams[i]);
        }
        for (BeamHyp &h : fin) beam_put(kv_pool(src), h.pages);
        fin.clear();
        live.clear();
    }
};

int32_t l2b_beam_search(l2b_ctx *src, int32_t token, int32_t pos, l2b_ctx *const *beams, int32_t n_beams,
                        int32_t n_steps, int32_t stop_on_bos, int32_t *out_tokens, int32_t *out_len,
                        float *out_logprob, int32_t *n_run) {
    if (!src) { g_create_error = "src is NULL"; return L2B_ERR_INVALID_ARG; }
    if (!beams || !out_tokens || !out_len || !out_logprob)
        return fail(src, L2B_ERR_INVALID_ARG, "beams, out_tokens, out_len or out_logprob is NULL");
    const int V = src->cfg.vocab_size;
    if (n_beams < 1 || n_beams > L2B_BEAM_MAX || 2 * n_beams > V)
        return fail(src, L2B_ERR_INVALID_ARG, "n_beams outside [1, L2B_BEAM_MAX], or 2 * n_beams > vocab_size");
    std::set<const l2b_ctx *> seen;
    for (int i = 0; i < n_beams; ++i) {
        const l2b_ctx *b = beams[i];
        if (!b) return fail(src, L2B_ERR_INVALID_ARG, "NULL beam");
        if (b == src) return fail(src, L2B_ERR_INVALID_ARG, "src among the beams");
        if (!seen.insert(b).second) return fail(src, L2B_ERR_INVALID_ARG, "the same beam twice");
        if (b->weights != src->weights) return fail(src, L2B_ERR_INVALID_ARG, "a beam of another model");
    }
    if (token < 0 || token >= V) return fail(src, L2B_ERR_INVALID_ARG, "token out of range");
    if (pos < 0 || pos >= src->cfg.seq_len) return fail(src, L2B_ERR_INVALID_ARG, "pos out of range");
    if (n_steps < 0) return fail(src, L2B_ERR_INVALID_ARG, "n_steps < 0");
    if (pos > src->n_appended) return fail(src, L2B_ERR_STATE, "pos past the positions src has appended");
    if (!src->paged)
        return fail(src, L2B_ERR_UNSUPPORTED,
                    "l2b_beam_search needs a paged model (L2B_KV_PAGED): on a contiguous cache each step's reorder "
                    "would copy O(pos) rows per beam");
    src->last_ms = 0.0f;
    src->last_launches = 0;
    if (n_run) *n_run = 0;
    if (n_steps == 0) {
        for (int i = 0; i < n_beams; ++i) { out_len[i] = 0; out_logprob[i] = 0.0f; }
        return L2B_OK;
    }
    l2b_ctx *lead = beams[0];
    L2B_CUDA(src, cudaSetDevice(src->device));
    int rc = pf_prepare(lead);
    if (!rc) rc = call_buf_reserve(lead, lead->call_ints, lead->call_ints_cap, (size_t)n_beams);
    if (!rc) rc = call_buf_reserve(lead, lead->call_cand, lead->call_cand_cap, (size_t)n_beams * 2 * n_beams);
    if (rc) { src->err = lead->err; return rc; }
    fill_ctl(lead, token, pos, 0, 1.0f, -1.0f);   // CTL_DONE = 0 for the batched kernels and the top-k kernel
    L2B_CUDA(src, cudaMemcpyAsync(lead->ctl, lead->h_ctl, CTL_HOST_WORDS * sizeof(int), cudaMemcpyHostToDevice, lead->stream));
    L2B_CUDA(src, cudaEventRecord(src->ev0, lead->stream));
    BeamSearch bs{src, lead, beams, n_beams, 2 * n_beams, pos, token, stop_on_bos != 0};
    rc = bs.run(n_steps);
    if (!rc) rc = bs.finish(n_steps, out_tokens, out_len, out_logprob);
    if (rc) {
        bs.abandon();
        return rc;
    }
    L2B_CUDA(src, cudaEventRecord(src->ev1, lead->stream));
    L2B_CUDA(src, cudaEventSynchronize(src->ev1));
    L2B_CUDA(src, cudaEventElapsedTime(&src->last_ms, src->ev0, src->ev1));
    src->last_launches = bs.launches;
    if (n_run) *n_run = bs.ran;
    return L2B_OK;
}

int32_t l2b_read_state(l2b_ctx *ctx, int32_t which, float *dst, uint64_t n, uint64_t *n_out) {
    if (!ctx || !dst) return L2B_ERR_INVALID_ARG;
    const void *src = nullptr;
    uint64_t cnt = 0;
    const uint64_t L = ctx->cfg.n_layers, S = ctx->cfg.seq_len;
    switch (which) {
    case 0: src = ctx->final_X ? ctx->final_X : ctx->X; cnt = ctx->dim; break;
    case 1: src = ctx->xb; cnt = ctx->q_loc; break;
    case 2: src = ctx->hb; cnt = ctx->hid_loc; break;
    case 3: src = ctx->q; cnt = ctx->q_loc; break;
    case 4: src = ctx->kcache; cnt = L * S * ctx->kv_loc; break;
    case 5: src = ctx->vcache; cnt = L * S * ctx->kv_loc; break;
    case 6: src = ctx->logits; cnt = ctx->cfg.vocab_size; break;
    default: return fail(ctx, L2B_ERR_INVALID_ARG, "unknown state id");
    }
    if (n < cnt) return fail(ctx, L2B_ERR_INVALID_ARG, "dst too small");
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    if (which != 4 && which != 5) {
        L2B_CUDA(ctx, cudaMemcpy(dst, src, cnt * sizeof(float), cudaMemcpyDeviceToHost));
        if (n_out) *n_out = cnt;
        return L2B_OK;
    }
    // The cache widened to fp32 layer by layer, each e4m3 layer with its own scale.  A paged cache is gathered
    // page by page into the contiguous layout, and rows of pages the context does not hold are 0.  A contiguous
    // cache of el-byte elements lands in the last el/4 of dst and is widened in place from the front: value i
    // is written to bytes [4i, 4i+4), below the unread elements at [cnt (4 - el) + el (i+1), ..).
    const int v = which == 5;
    const uint64_t kvl = ctx->kv_loc, P = KV_PAGE_ROWS;
    return with_kv_elem(ctx->kvfmt, [&](auto e) -> int32_t {
        const size_t el = sizeof(typename decltype(e)::type);
        auto widen = [&](const unsigned char *from, uint64_t l, uint64_t row0, uint64_t rows) {
            kv_widen(e, from, dst + (l * S + row0) * kvl, rows * kvl, kv_scaled(ctx->kvfmt) ? ctx->weights->kv_scale_h[2 * l + v] : 1.0f);
        };
        if (ctx->paged) {
            memset(dst, 0, cnt * sizeof(float));
            std::vector<unsigned char> page(kv_page_bytes(ctx));
            for (int j = 0; j < ctx->n_pages; ++j) {
                if (!ctx->pages[j]) continue;
                L2B_CUDA(ctx, cudaMemcpy(page.data(), ctx->pages[j], page.size(), cudaMemcpyDeviceToHost));
                for (uint64_t l = 0; l < L; ++l) widen(page.data() + (2 * l + v) * P * kvl * el, l, j * P, std::min<uint64_t>(P, S - j * P));
            }
        } else {
            unsigned char *h = reinterpret_cast<unsigned char *>(dst) + cnt * (4 - el);
            L2B_CUDA(ctx, cudaMemcpy(h, src, cnt * el, cudaMemcpyDeviceToHost));
            for (uint64_t l = 0; l < L; ++l) widen(h + l * S * kvl * el, l, 0, S);
        }
        if (n_out) *n_out = cnt;
        return L2B_OK;
    });
}

int32_t l2b_last_timing(const l2b_ctx *ctx, float *device_ms, int32_t *kernel_launches) {
    if (!ctx) return L2B_ERR_INVALID_ARG;
    if (device_ms) *device_ms = ctx->last_ms;
    if (kernel_launches) *kernel_launches = ctx->last_launches;
    return L2B_OK;
}

int32_t l2b_load_stats(const l2b_ctx *ctx, double *upload_ms, uint64_t *upload_bytes) {
    if (!ctx) return L2B_ERR_INVALID_ARG;
    if (upload_ms) *upload_ms = ctx->load_ms;
    if (upload_bytes) *upload_bytes = ctx->load_bytes;
    return L2B_OK;
}

int32_t l2b_profile_step(l2b_ctx *ctx, int32_t token, int32_t pos, l2b_kernel_time *out, int32_t cap,
                         int32_t *n_out) {
    int rc = check_step_args(ctx, token, pos);
    if (rc) return rc;
    if (!out || !n_out || cap <= 0) return fail(ctx, L2B_ERR_INVALID_ARG, "bad profile arguments");
    std::vector<l2b_ctx *> ranks = locals(ctx);
    KvCall kv;
    rc = kv.reserve(ctx, {{ctx, pos, pos + 1}});
    if (rc) return rc;
    if (pos + 1 > ctx->n_appended) ctx->n_appended = pos + 1;   // attention bytes use this
    const int saved_appended = ctx->n_appended;
    cudaEvent_t last = nullptr;
    for (l2b_ctx *c : ranks) {
        L2B_CUDA(ctx, cudaSetDevice(c->device));
        c->n_appended = pos + 1;
        fill_ctl(c, token, pos, 0, 1.0f, -1.0f);
        L2B_CUDA(ctx, cudaMemcpyAsync(c->ctl, c->h_ctl, CTL_HOST_WORDS * sizeof(int), cudaMemcpyHostToDevice, c->stream));
        c->profiling = (c == ctx);
        c->prof_ev.clear();
        c->prof_rec.clear();
        int r2 = enqueue_step(c, c->stream, MODE_LOGITS);
        c->profiling = false;
        if (r2 && rc == L2B_OK) { rc = r2; ctx->err = c->err; }
        if (c == ctx && rc == L2B_OK) {
            if (cudaEventCreate(&last) != cudaSuccess || cudaEventRecord(last, c->stream) != cudaSuccess)
                rc = fail(ctx, L2B_ERR_CUDA, "event record failed");
        }
        cudaMemcpyAsync(c->h_ctl + CTL_WORDS, c->ctl, CTL_WORDS * sizeof(int), cudaMemcpyDeviceToHost, c->stream);
    }
    ctx->n_appended = saved_appended;
    {
        int r2 = finish_call(ranks.data(), ranks.size());
        if (rc == L2B_OK) rc = r2;
    }
    cudaSetDevice(ctx->device);
    const int n = (int)ctx->prof_rec.size();
    if (rc == L2B_OK) {
        for (int i = 0; i < n; ++i) {
            cudaEvent_t b = (i + 1 < n) ? ctx->prof_ev[i + 1] : last;
            float ms = 0.0f;
            cudaEventElapsedTime(&ms, ctx->prof_ev[i], b);
            ctx->prof_rec[i].ms = ms;
            if (i < cap) out[i] = ctx->prof_rec[i];
        }
        *n_out = n;
    }
    for (cudaEvent_t e : ctx->prof_ev) cudaEventDestroy(e);
    if (last) cudaEventDestroy(last);
    ctx->prof_ev.clear();
    return rc;
}

// debug: copy the in-kernel timeline of the last step (L2B_TRACE=1) to the host
int32_t l2b_debug_trace(l2b_ctx *ctx, unsigned long long *dst, uint64_t cap_words, uint64_t *n_words) {
    if (!ctx || !dst) return L2B_ERR_INVALID_ARG;
    if (!ctx->trace) return fail(ctx, L2B_ERR_STATE, "tracing not enabled (L2B_TRACE=1)");
    const uint64_t n = (uint64_t)ctx->trace_launches * TRACE_MAX_CTAS * TRACE_SLOTS;
    if (cap_words < n) return fail(ctx, L2B_ERR_INVALID_ARG, "dst too small");
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    L2B_CUDA(ctx, cudaMemcpy(dst, ctx->trace, n * 8, cudaMemcpyDeviceToHost));
    if (n_words) *n_words = n;
    return L2B_OK;
}

int32_t l2b_step_bytes(const l2b_ctx *ctx, int32_t pos, uint64_t *weight_bytes, uint64_t *kv_bytes) {
    if (!ctx) return L2B_ERR_INVALID_ARG;
    const uint64_t dim = ctx->dim, L = ctx->cfg.n_layers;
    // SURVEY.md 8d: every weight touched once per token (+ the embedding row), this rank's shard.
    // Matrices count w_elem bytes per stored element (bf16 rows with their padding), gains 4.
    const uint64_t ld_dim = w_ld(ctx, dim), ld_q = w_ld(ctx, ctx->q_loc), ld_hid = w_ld(ctx, ctx->hid_loc);
    const uint64_t mat = L * ((uint64_t)ctx->q_loc * ld_dim + 2ull * ctx->kv_loc * ld_dim + dim * ld_q +
                              2ull * ctx->hid_loc * ld_dim + dim * ld_hid) +
                         ld_dim + (uint64_t)ctx->vocab_loc * ld_dim;
    if (weight_bytes) *weight_bytes = w_elem(ctx) * mat + 4 * (L * 2 * dim);
    if (kv_bytes) *kv_bytes = kv_elem(ctx) * L * 2 * ctx->kv_loc * (uint64_t)(pos + 1);
    return L2B_OK;
}

int32_t l2b_comm_unique_id(uint8_t id[128]) {
    if (!id) return L2B_ERR_INVALID_ARG;
    std::string e;
    if (!nccl_load(&e)) { g_create_error = e; return L2B_ERR_COMM; }
    ncclUniqueId u;
    if (g_nccl.GetUniqueId(&u) != ncclSuccess) { g_create_error = "ncclGetUniqueId failed"; return L2B_ERR_COMM; }
    memcpy(id, &u, 128);
    return L2B_OK;
}

// ---- synthetic generator, host mirror ------------------------------------------------------
void l2b_synth_fill_host(float *dst, uint64_t first, uint64_t count, uint64_t tensor_seed, double mean,
                         double sigma, float lo, float hi) {
    const double scale = sigma * kSynthInvStd;
    for (uint64_t j = 0; j < count; ++j) {
        const int32_t s = synth_irwin_hall(tensor_seed, first + j);
        volatile double prod = (double)s * scale;   // no a*b+c contraction
        float v = (float)(prod + mean);
        v = fminf(fmaxf(v, lo), hi);
        dst[j] = v;
    }
}

int32_t l2b_synth_checkpoint_host(const l2b_config *cfg, uint64_t seed, float *data, uint64_t n_floats) {
    if (!cfg || !data) return L2B_ERR_INVALID_ARG;
    if (n_floats < checkpoint_floats(cfg)) return L2B_ERR_INVALID_ARG;
    const uint64_t dim = cfg->dim, hid = cfg->hidden_dim, L = cfg->n_layers, V = cfg->vocab_size, S = cfg->seq_len;
    const uint64_t hs = dim / cfg->n_heads, kvd = hs * cfg->n_kv_heads;
    const double sd = sqrt(288.0 / (double)dim), sh = sqrt(768.0 / (double)hid);
    const float BIG = 3.0e38f;
    float *p = data;
    auto T = [&](int id, uint64_t count, double mean, double sigma, float lo, float hi) {
        l2b_synth_fill_host(p, 0, count, mix64(seed * 1000003ull + (uint64_t)id), mean, sigma, lo, hi);
        p += count;
    };
    T(1, V * dim, 0.0, 0.04, -BIG, BIG);
    T(2, L * dim, 1.35, 0.35, 0.25f, 2.4f);
    T(3, L * dim * dim, 0.0, 0.04 * sd, -BIG, BIG);
    T(4, L * kvd * dim, 0.0, 0.04 * sd, -BIG, BIG);
    T(5, L * kvd * dim, 0.0, 0.02 * sd, -BIG, BIG);
    T(6, L * dim * dim, 0.0, 0.02 * sd, -BIG, BIG);
    T(7, L * dim, 1.35, 0.35, 0.25f, 2.4f);
    T(8, L * hid * dim, 0.0, 0.026 * sd, -BIG, BIG);
    T(9, L * dim * hid, 0.0, 0.026 * sh, -BIG, BIG);
    T(10, L * hid * dim, 0.0, 0.026 * sd, -BIG, BIG);
    T(11, dim, 7.1, 0.6, 3.0f, 10.0f);
    memset(p, 0, sizeof(float) * 2 * (S * hs / 2));
    p += 2 * (S * hs / 2);
    if (!cfg->shared_weights) T(14, V * dim, 0.0, 0.04, -BIG, BIG);
    return L2B_OK;
}

// ---- single ops with host buffers (unit-test surface) ----------------------------------------
namespace {
struct OpScope {
    int rc = L2B_OK;
    std::vector<void *> bufs;
    explicit OpScope(int device) {
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); rc = L2B_ERR_NO_DEVICE; g_create_error = "no CUDA device"; return; }
        if (device < 0 || device >= ndev) { rc = L2B_ERR_INVALID_ARG; g_create_error = "device out of range"; return; }
        if (cudaSetDevice(device) != cudaSuccess) { rc = L2B_ERR_CUDA; g_create_error = "cudaSetDevice failed"; }
    }
    float *up(const float *h, size_t n) {
        if (rc) return nullptr;
        void *d = nullptr;
        if (cudaMalloc(&d, (n ? n : 1) * sizeof(float)) != cudaSuccess) { rc = L2B_ERR_OOM; g_create_error = "cudaMalloc failed"; return nullptr; }
        bufs.push_back(d);
        if (h && cudaMemcpy(d, h, n * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) { rc = L2B_ERR_CUDA; g_create_error = "H2D failed"; }
        return (float *)d;
    }
    void down(float *h, const float *d, size_t n) {
        if (rc) return;
        cudaError_t e = cudaDeviceSynchronize();
        if (e == cudaSuccess) e = cudaMemcpy(h, d, n * sizeof(float), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { rc = L2B_ERR_CUDA; g_create_error = std::string("op failed: ") + cudaGetErrorString(e); }
    }
    ~OpScope() { for (void *p : bufs) cudaFree(p); }
};
}  // namespace

// W . rmsnorm(x, gamma) (gamma NULL => W . x), optionally accumulated into resid_inout, through a
// chosen GEMV kernel flavour: the fused prologue / residual epilogue of the hot path in isolation
int32_t l2b_op_fused_matmul(int32_t device, float *xout, const float *x, const float *gamma, const float *w,
                            float *resid_inout, int32_t d, int32_t n, int32_t kernel) {
    if ((!xout && !resid_inout) || !x || !w || d <= 0 || n <= 0 || kernel < 0 || kernel > 3) return L2B_ERR_INVALID_ARG;
    if (n % 4) { g_create_error = "n must be a multiple of 4"; return L2B_ERR_UNSUPPORTED; }
    OpScope s(device);
    float *dx = s.up(x, n), *dw = s.up(w, (size_t)d * n), *dg = gamma ? s.up(gamma, n) : nullptr;
    float *dout = s.up(resid_inout ? resid_inout : nullptr, d);
    int *ctl = (int *)s.up(nullptr, CTL_WORDS);
    if (s.rc) return s.rc;
    cudaMemset(ctl, 0, CTL_WORDS * sizeof(int));
    l2b_ctx tmp;   // only for launch_gemv's bookkeeping
    tmp.device = device;
    tmp.force_kernel = kernel;
    cudaDeviceProp prop{};
    cudaGetDeviceProperties(&prop, device);
    tmp.num_sms = prop.multiProcessorCount;
    GemvParams p{};
    p.ctl = ctl; p.n = n; p.x_in = dx; p.gamma = dg; p.w0 = dw; p.total_rows = d; p.rows0 = d; p.out0 = dout;
    int rc = launch_gemv(&tmp, resid_inout ? EPI_RESID : EPI_STORE, p, 0);
    if (rc) { g_create_error = tmp.err; return rc; }
    s.down(resid_inout ? resid_inout : xout, dout, d);
    return s.rc;
}

int32_t l2b_op_matmul(int32_t device, float *xout, const float *x, const float *w, int32_t d, int32_t n) {
    if (!xout || !x || !w || d <= 0 || n <= 0) return L2B_ERR_INVALID_ARG;   // asserts :534-536
    if (n % 4 == 0) return l2b_op_fused_matmul(device, xout, x, nullptr, w, nullptr, d, n, 0);
    OpScope s(device);
    float *dx = s.up(x, n), *dw = s.up(w, (size_t)d * n), *dout = s.up(nullptr, d);
    if (s.rc) return s.rc;
    int blocks = (d + NWARP - 1) / NWARP;
    gemv_scalar_kernel<<<blocks, NT>>>(dout, dx, dw, d, n);
    s.down(xout, dout, d);
    return s.rc;
}

int32_t l2b_op_rmsnorm(int32_t device, float *o, const float *x, const float *w, int32_t n) {
    if (!o || !x || !w || n <= 0) return L2B_ERR_INVALID_ARG;
    OpScope s(device);
    float *dx = s.up(x, n), *dw = s.up(w, n), *dout = s.up(nullptr, n);
    if (s.rc) return s.rc;
    rmsnorm_kernel<<<1, NT>>>(dout, dx, dw, n);
    s.down(o, dout, n);
    return s.rc;
}

int32_t l2b_op_softmax(int32_t device, float *x, int32_t n) {
    if (!x || n <= 0) return L2B_ERR_INVALID_ARG;   // assert :688
    OpScope s(device);
    float *dx = s.up(x, n);
    if (s.rc) return s.rc;
    softmax_kernel<<<1, NT>>>(dx, n);
    s.down(x, dx, n);
    return s.rc;
}

int32_t l2b_op_weighted_sum_rows(int32_t device, float *xout, int32_t out_len, const float *rows,
                                 int32_t row_stride, const float *weights, int32_t n_weights) {
    if (!xout || !rows || !weights || out_len <= 0 || n_weights <= 0 || row_stride < out_len)
        return L2B_ERR_INVALID_ARG;   // asserts :658-661
    OpScope s(device);
    const size_t nrows = (size_t)(n_weights - 1) * row_stride + out_len;
    float *dr = s.up(rows, nrows), *dw = s.up(weights, n_weights), *dout = s.up(nullptr, out_len);
    if (s.rc) return s.rc;
    weighted_rows_kernel<<<(out_len + NT - 1) / NT, NT>>>(dout, out_len, dr, row_stride, dw, n_weights);
    s.down(xout, dout, out_len);
    return s.rc;
}

int32_t l2b_op_attention_head(int32_t device, float *out, const float *q, const float *keys,
                              const float *values, int32_t head_size, int32_t kv_stride, int32_t n_pos) {
    if (!out || !q || !keys || !values || head_size <= 0 || n_pos <= 0 || kv_stride < head_size)
        return L2B_ERR_INVALID_ARG;
    if (head_size % 4 || kv_stride % 4 || head_size > NT) { g_create_error = "head_size/kv_stride must be multiples of 4 and head_size <= 256"; return L2B_ERR_UNSUPPORTED; }
    OpScope s(device);
    const size_t nkv = (size_t)n_pos * kv_stride;
    float *dq = s.up(q, head_size), *dk = s.up(keys, nkv), *dv = s.up(values, nkv), *dout = s.up(nullptr, head_size);
    const int nsplit = n_pos > 256 ? 4 : 1;
    float *po = s.up(nullptr, (size_t)nsplit * head_size), *pml = s.up(nullptr, (size_t)nsplit * 2);
    unsigned int *cnt = (unsigned int *)s.up(nullptr, 1);
    int *ctl = (int *)s.up(nullptr, CTL_WORDS);
    if (s.rc) return s.rc;
    int hctl[CTL_WORDS] = {0, n_pos - 1};
    cudaMemcpy(ctl, hctl, sizeof hctl, cudaMemcpyHostToDevice);
    cudaMemset(cnt, 0, sizeof(unsigned int));
    AttnParams a{};
    a.ctl = ctl; a.q = dq; a.kcache = dk; a.vcache = dv; a.xb = dout; a.part_o = po; a.part_ml = pml;
    a.counters = cnt; a.head_size = head_size; a.kv_dim = kv_stride; a.kv_mul = 1; a.nsplit = nsplit;
    a.min_chunk = 64;
    a.seq_len = n_pos;
    int cap = (n_pos + nsplit - 1) / nsplit;
    if (cap < 64) cap = 64;
    const int G = NT / (head_size / 4);
    const size_t smem = ((size_t)G * head_size + cap) * sizeof(float);
    if (smem > (size_t)kMaxDynSmem) { g_create_error = "n_pos too large"; return L2B_ERR_UNSUPPORTED; }
    cudaFuncSetAttribute(attention_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
    {
        const char *enva = getenv("L2B_ATTN");
        size_t smem2 = smem;
        attn_fn fn = pick_attention(head_size, !(enva && strcmp(enva, "3pass") == 0), &smem2);
        fn<<<dim3(1, nsplit), NT, smem2>>>(a, AttnBatch{});
    }
    s.down(out, dout, head_size);
    return s.rc;
}

// log softmax(logits)[target] alone (logprob_batch_kernel, one row) on host logits: unit-test surface
int32_t l2b_op_logprob(int32_t device, const float *logits, int32_t n, int32_t target, float *logprob) {
    if (!logits || !logprob || n < 1 || target < 0 || target >= n) return L2B_ERR_INVALID_ARG;
    OpScope s(device);
    float *dl = s.up(logits, n), *dlp = s.up(nullptr, 1);
    int *ctl = (int *)s.up(nullptr, CTL_WORDS), *dt = (int *)s.up(nullptr, 1), *dg = (int *)s.up(nullptr, 1);
    unsigned long long *amax = (unsigned long long *)s.up(nullptr, 2);
    if (s.rc) return s.rc;
    cudaMemset(ctl, 0, CTL_WORDS * sizeof(int));
    cudaMemset(amax, 0, sizeof(unsigned long long));
    cudaMemcpy(dt, &target, sizeof(int), cudaMemcpyHostToDevice);
    LogprobBatchParams p{ctl, dl, n, dt, amax, dlp, dg};
    logprob_batch_kernel<<<1, LOGPROB_THREADS>>>(p);
    s.down(logprob, dlp, 1);
    return s.rc;
}

// the k best log softmax(logits)[i] alone (logprob_topk_batch_kernel, one row): unit-test surface
int32_t l2b_op_logprob_topk(int32_t device, const float *logits, int32_t n, int32_t k, l2b_prob_index *out) {
    if (!logits || !out || n < 1 || k < 1 || k > n || k > 2 * L2B_BEAM_MAX) return L2B_ERR_INVALID_ARG;
    static_assert(2 * L2B_BEAM_MAX == TOPK_MAX, "the top-k kernel keeps 2 * L2B_BEAM_MAX keys per thread");
    static_assert(sizeof(l2b_prob_index) == sizeof(ProbIndex), "candidate layout");
    OpScope s(device);
    float *dl = s.up(logits, n), *dout = s.up(nullptr, (size_t)2 * k);
    int *ctl = (int *)s.up(nullptr, CTL_WORDS);
    if (s.rc) return s.rc;
    cudaMemset(ctl, 0, CTL_WORDS * sizeof(int));
    LogprobTopkParams p{ctl, dl, n, n, k, reinterpret_cast<ProbIndex *>(dout)};
    logprob_topk_batch_kernel<<<1, LOGPROB_THREADS>>>(p);
    s.down(reinterpret_cast<float *>(out), dout, (size_t)2 * k);
    return s.rc;
}

// sampler preparation alone (src/main.zig:1005-1008, :761-768) on host logits: unit-test surface
int32_t l2b_op_sample_prep(int32_t device, float *logits_inout, int32_t n, float temperature, float top_p,
                           l2b_prob_index *cand, int32_t cand_cap, int32_t *n_cand) {
    if (!logits_inout || n <= 1 || !(temperature > 0.0f) || !n_cand) return L2B_ERR_INVALID_ARG;
    OpScope s(device);
    float *dl = s.up(logits_inout, n);
    int *ctl = (int *)s.up(nullptr, CTL_WORDS);
    ProbIndex *dc = (ProbIndex *)s.up(nullptr, (size_t)2 * (cand_cap > 0 ? cand_cap : 1));
    int *dn = (int *)s.up(nullptr, 1);
    if (s.rc) return s.rc;
    const bool filter = (top_p != 0.0f && top_p != 1.0f);
    const float tp = filter ? top_p : -1.0f;
    int hctl[CTL_WORDS] = {0};
    memcpy(&hctl[CTL_TEMP], &temperature, sizeof(float));
    memcpy(&hctl[CTL_TOPP], &tp, sizeof(float));
    cudaMemcpy(ctl, hctl, sizeof hctl, cudaMemcpyHostToDevice);
    cudaMemset(dn, 0, sizeof(int));
    sample_prep_kernel<<<1, SAMP_THREADS>>>(dl, n, ctl, dc, cand_cap, dn);
    s.down(logits_inout, dl, n);
    if (s.rc) return s.rc;
    int hn = 0;
    cudaMemcpy(&hn, dn, sizeof(int), cudaMemcpyDeviceToHost);
    *n_cand = hn;
    if (filter && cand && hn > 0) {
        const int m = hn < cand_cap ? hn : cand_cap;
        cudaMemcpy(cand, dc, (size_t)m * sizeof(ProbIndex), cudaMemcpyDeviceToHost);
    }
    return s.rc;
}

}  // extern "C"
