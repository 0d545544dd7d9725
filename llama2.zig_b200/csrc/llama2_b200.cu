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
#include <chrono>
#include <set>
#include <string>
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
struct SharedWeights {
    int refs = 1;
    std::vector<void *> owned;
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
    float *emb = nullptr, *rms_att = nullptr, *rms_ffn = nullptr, *rms_final = nullptr;
    float *wq = nullptr, *wk = nullptr, *wv = nullptr, *wo = nullptr;
    float *w1 = nullptr, *w2 = nullptr, *w3 = nullptr, *wcls = nullptr;
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
    int *pf_tokens = nullptr;
    bool pf_ready = false, pf_ok = false;
    int *gb_ints = nullptr;                  // l2b_generate_argmax_batch on the batched path: its per-call
    size_t gb_cap = 0;                       // session and token arrays (ints), grown on demand
    int attn_R = 1;                          // CTAs per head cluster of attn_wo_kernel
    float *delta = nullptr;                  // L2B_TP=nccl baseline only: partial rows before the NCCL all-reduce
    float *q = nullptr, *xb = nullptr, *hb = nullptr, *logits = nullptr, *logits_loc = nullptr;
    float *kcache = nullptr, *vcache = nullptr;     // (L, seq_len, kv_loc)
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
    int tma_ctas_per_sm = 1;                 // ring CTAs one SM's shared memory is split for (L2B_TMA_CTAS)
    size_t smem_per_sm = 0, smem_reserved = 0;   // shared memory per SM, and reserved by the system per block
    int tma_stages = 0;                      // 0 = auto; else forced ring depth
    int tma_prefill = 0;                     // stages in flight before the dependency wait; 0 = the whole ring (L2B_TMA_PREFILL)
    bool big_kernel_tma = true;              // bandwidth-bound GEMVs: TMA-ring kernel (false: register-fed 8-row kernel)
    long long gemv8_min_bytes = 8ll << 20;   // >= this many weight bytes (and n >= big_min_n): streaming kernel; -1 = never
    int big_min_n = 1024;                    // measured r02: at n = 768 the TMA ring (192 of 256 columns per stage) loses to the latency kernel
    int tpr_min_tiles_per_sm = 0;            // > 0: shrink threads-per-row while the grid still has this many tiles per SM (L2B_TPR_TILES)
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
int upload(l2b_ctx *ctx, float *dst, const float *src, uint64_t rows, uint64_t cols, uint64_t src_pitch) {
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
    const uint64_t row_bytes = cols * sizeof(float);
    const bool dense = (src_pitch == cols);
    const uint64_t total = rows * row_bytes;
    uint64_t done = 0;                       // bytes of the dense destination already issued
    while (done < total) {
        const int b = ctx->stage_next;
        ctx->stage_next ^= 1;
        L2B_CUDA(ctx, cudaEventSynchronize(ctx->stage_ev[b]));   // previous DMA out of this buffer finished
        uint64_t chunk = total - done < ctx->stage_bytes ? total - done : ctx->stage_bytes;
        if (!dense) {
            // whole rows only (a chunk never splits a row of a sharded window)
            uint64_t r = chunk / row_bytes;
            if (r == 0) return fail(ctx, L2B_ERR_UNSUPPORTED, "row larger than the upload staging buffer");
            chunk = r * row_bytes;
            const uint64_t row0 = done / row_bytes;
            for (uint64_t i = 0; i < r; ++i)
                memcpy(ctx->stage[b] + i * row_bytes, src + (row0 + i) * src_pitch, row_bytes);
        } else {
            memcpy(ctx->stage[b], reinterpret_cast<const unsigned char *>(src) + done, chunk);
        }
        L2B_CUDA(ctx, cudaMemcpyAsync(reinterpret_cast<unsigned char *>(dst) + done, ctx->stage[b], chunk,
                                      cudaMemcpyHostToDevice, ctx->stream));
        L2B_CUDA(ctx, cudaEventRecord(ctx->stage_ev[b], ctx->stream));
        done += chunk;
    }
    ctx->load_bytes += total;
    return L2B_OK;
}

int materialize(l2b_ctx *ctx, float **dptr, const Source &src, uint64_t payload_off, int tensor_id,
                uint64_t L, uint64_t rows, uint64_t cols, ShardMode mode, Dist dist) {
    const uint64_t g = ctx->world, r = ctx->rank;
    const uint64_t rows_loc = (mode == SH_ROWS) ? rows / g : rows;
    const uint64_t cols_loc = (mode == SH_COLS) ? cols / g : cols;
    const uint64_t row0 = (mode == SH_ROWS) ? r * rows_loc : 0;
    const uint64_t col0 = (mode == SH_COLS) ? r * cols_loc : 0;
    int rc = dev_alloc(ctx, dptr, L * rows_loc * cols_loc, &ctx->weights->owned);
    if (rc) return rc;
    const uint64_t tensor_seed = mix64(src.seed * 1000003ull + (uint64_t)tensor_id);
    const bool whole = (rows_loc == rows && cols_loc == cols);
    const uint64_t nl = whole ? 1 : L;            // one shot when nothing is cut
    const uint64_t rr = whole ? L * rows : rows_loc;
    for (uint64_t l = 0; l < nl; ++l) {
        float *dst = *dptr + l * rows_loc * cols_loc;
        const uint64_t first = l * rows * cols + row0 * cols + col0;
        if (src.host) {
            rc = upload(ctx, dst, src.host + payload_off + first, rr, cols_loc, cols);
            if (rc) return rc;
        } else {
            const uint64_t total = rr * cols_loc;
            int blocks = (int)((total + 255) / 256 < (uint64_t)(ctx->num_sms * 16)
                                   ? (total + 255) / 256
                                   : (uint64_t)(ctx->num_sms * 16));
            if (blocks < 1) blocks = 1;
            synth_fill_kernel<<<blocks, 256, 0, ctx->stream>>>(dst, rr, cols_loc, first, cols, tensor_seed,
                                                               dist.mean, dist.sigma * kSynthInvStd,
                                                               dist.lo, dist.hi);
            L2B_CUDA(ctx, cudaGetLastError());
        }
    }
    return L2B_OK;
}

// ---- GEMV launch ---------------------------------------------------------------------------
typedef void (*gemv_fn)(const GemvParams);

template <int EPI>
gemv_fn gemv_pick(int tpr) {
    switch (tpr) {
    case 8: return gemv_kernel<8, EPI>;
    case 16: return gemv_kernel<16, EPI>;
    case 32: return gemv_kernel<32, EPI>;
    case 64: return gemv_kernel<64, EPI>;
    case 128: return gemv_kernel<128, EPI>;
    default: return gemv_kernel<256, EPI>;
    }
}
gemv_fn gemv_pick(int epi, int tpr) {
    switch (epi) {
    case EPI_XCHG: return gemv_pick<EPI_XCHG>(tpr);
    case EPI_RESID: return gemv_pick<EPI_RESID>(tpr);
    case EPI_STORE: return gemv_pick<EPI_STORE>(tpr);
    case EPI_ARGMAX: return gemv_pick<EPI_ARGMAX>(tpr);
    case EPI_QKV: return gemv_pick<EPI_QKV>(tpr);
    default: return gemv_pick<EPI_SILU>(tpr);
    }
}

constexpr int kMaxDynSmem = 200 * 1024;
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

gemv_fn gemv_tma_pick(int epi) {
    switch (epi) {
    case EPI_XCHG: return gemv_tma_kernel<EPI_XCHG>;
    case EPI_RESID: return gemv_tma_kernel<EPI_RESID>;
    case EPI_STORE: return gemv_tma_kernel<EPI_STORE>;
    case EPI_ARGMAX: return gemv_tma_kernel<EPI_ARGMAX>;
    case EPI_QKV: return gemv_tma_kernel<EPI_QKV>;
    default: return gemv_tma_kernel<EPI_SILU>;
    }
}

gemv_fn gemv8_pick(int epi) {
    switch (epi) {
    case EPI_XCHG: return gemv8_kernel<EPI_XCHG>;
    case EPI_RESID: return gemv8_kernel<EPI_RESID>;
    case EPI_STORE: return gemv8_kernel<EPI_STORE>;
    case EPI_ARGMAX: return gemv8_kernel<EPI_ARGMAX>;
    case EPI_QKV: return gemv8_kernel<EPI_QKV>;
    default: return gemv8_kernel<EPI_SILU>;
    }
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

// Depth of gemv_tma_kernel's ring next to xbytes of x when `ctas` ring CTAs are to share one SM:
// each gets 1/ctas of the SM's shared memory, less the per-block reservation and its static
// shared memory, so any two ring kernels sized for the same split fit on one SM together.
int tma_ring_slots(const l2b_ctx *ctx, int ctas, size_t static_bytes, size_t xbytes) {
    const size_t share = ctx->smem_per_sm / (size_t)ctas;
    const size_t used = ctx->smem_reserved + static_bytes;
    size_t budget = share > used ? share - used : 0;
    if (budget > (size_t)kMaxSmemOptin) budget = kMaxSmemOptin;
    return tma_ring_stages(budget, xbytes, (size_t)TmaRing<TMA_SLOT_ROWS>::SLOT_FLOATS * 4, TMA_MAX_STAGES);
}

int launch_gemv(l2b_ctx *ctx, int epi, const GemvParams &p, cudaStream_t st, const char *name = "gemv",
                int layer = -1) {
    {
        int prc = prof_mark(ctx, name, layer, (uint64_t)p.total_rows * p.n * 4ull, st);
        if (prc) return prc;
    }
    const size_t xbytes = (size_t)p.n * 4 * (1 + (p.gamma ? 1 : 0) + (p.parts ? 1 : 0));
    // bandwidth-bound shapes take the TMA-ring kernel (or the register-fed 8-row kernel when
    // L2B_GEMV_BIG=ldg), latency-bound ones the fine-grained kernel
    bool big = ctx->gemv8_min_bytes >= 0 && p.n >= ctx->big_min_n &&
               (uint64_t)p.total_rows * p.n * 4ull >= (uint64_t)ctx->gemv8_min_bytes;
    if (ctx->force_kernel == 1) big = false;
    if (ctx->force_kernel >= 2) big = true;
    // TMA-ring kernel: only x is staged in shared memory, the rest of the CTA's share of the SM is a
    // ring of 16 KB slots.  The grid has one ring CTA per SM; the ring is sized for tma_ctas_per_sm
    // CTAs per SM (L2B_TMA_CTAS).  With 2, the free place is taken by the next kernel's CTA, which
    // fills its own ring before its dependency wait while this one drains; but a half-SM ring keeps
    // too few bytes in flight, and on llama2-7B the whole-SM ring (13 slots) is faster (measured on
    // an H100 SXM at 700 W: DESIGN.md §4.1).  An x too wide for a ring of 2 slots in that share
    // takes the whole SM.
    const size_t slot_bytes = (size_t)TmaRing<TMA_SLOT_ROWS>::SLOT_FLOATS * 4;
    const size_t xonly = (size_t)p.n * 4;
    gemv_fn tma_fn = gemv_tma_pick(epi);
    int nstage = 0;
    if (big && ctx->big_kernel_tma) {
        cudaFuncAttributes fa{};
        L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)tma_fn));
        nstage = tma_ring_slots(ctx, ctx->tma_ctas_per_sm, fa.sharedSizeBytes, xonly);
        if (nstage < 2) nstage = tma_ring_slots(ctx, 1, fa.sharedSizeBytes, xonly);
    }
    if (ctx->tma_stages > 0) nstage = ctx->tma_stages < TMA_MAX_STAGES ? ctx->tma_stages : TMA_MAX_STAGES;
    const bool fused_ok = !p.gamma || p.n <= TMA_MAXV * TMA_PRO_THREADS * 4;   // register slices of the rmsnorm gain
    if (p.parts && big) return fail(ctx, L2B_ERR_UNSUPPORTED, "partial-vector prologue is only in the latency kernel");
    bool tma = big && ctx->big_kernel_tma && nstage >= 2 && fused_ok && p.head_size <= 256 &&
               (size_t)nstage * slot_bytes + xonly <= (size_t)kMaxSmemOptin;
    if (ctx->force_kernel == 2) tma = false;
    if (ctx->force_kernel == 3 && !tma) return fail(ctx, L2B_ERR_UNSUPPORTED, "shape does not fit the TMA-ring kernel");
    const size_t smem = tma ? (size_t)nstage * slot_bytes + xonly : xbytes;
    if (smem > (size_t)kMaxSmemOptin) return fail(ctx, L2B_ERR_UNSUPPORTED, "activation vector too large for shared memory");
    // hard invariant of the ring kernel, whatever the budget arithmetic above decided
    if (tma && nstage < 2) return fail(ctx, L2B_ERR_UNSUPPORTED, "TMA ring of fewer than 2 stages");
    int tpr = gemv_tpr(p.n);
    // many-row matrices (the classifier): fewer threads per row = more 128-bit loads in flight per
    // thread and fewer shuffle steps per row, as long as the grid still covers the SMs
    while (ctx->tpr_min_tiles_per_sm > 0 && tpr > 8 &&
           (p.total_rows + (NT / (tpr / 2)) * GEMV_R - 1) / ((NT / (tpr / 2)) * GEMV_R) >= ctx->tpr_min_tiles_per_sm * ctx->num_sms)
        tpr /= 2;
    gemv_fn fn = tma ? tma_fn : big ? gemv8_pick(epi) : gemv_pick(epi, tpr);
    if (!ctx->attr_done.count((const void *)fn)) {
        L2B_CUDA(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemOptin));
        ctx->attr_done.insert((const void *)fn);
    }
    const int threads = tma ? TMA_THREADS : NT;
    int occ = 0;
    L2B_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, threads, smem));
    if (occ < 1) occ = 1;
    if (tma) occ = 1;                        // one ring CTA per SM: the other places are the successor's
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

// flash-decoding form when head_size/4 splits into 1..8 float4 per lane, else the 3-pass kernel
typedef void (*attn_fn)(const AttnParams, const AttnBatch);
attn_fn pick_attention(int head_size, bool flash, size_t *smem) {
    const int hs4 = head_size / 4;
    const int lpr = (hs4 % 8 == 0) ? 8 : (hs4 % 4 == 0) ? 4 : (hs4 % 2 == 0) ? 2 : 1;
    const int nf = hs4 / lpr;
    attn_fn f2 = nullptr;
    if (flash) {
        switch (nf) {
        case 1: f2 = attention_flash_kernel<1>; break;
        case 2: f2 = attention_flash_kernel<2>; break;
        case 3: f2 = attention_flash_kernel<3>; break;
        case 4: f2 = attention_flash_kernel<4>; break;
        case 5: f2 = attention_flash_kernel<5>; break;
        case 6: f2 = attention_flash_kernel<6>; break;
        case 8: f2 = attention_flash_kernel<8>; break;
        default: break;
        }
    }
    if (!f2) return attention_kernel;
    const int ng = NWARP * (32 / lpr);
    *smem = ((size_t)ng * head_size + 3 * (size_t)ng) * sizeof(float);
    return f2;
}

typedef void (*attn_wo_fn)(const AttnWoParams);
attn_wo_fn pick_attn_wo(int head_size, size_t *smem) {
    const int hs4 = head_size / 4;
    const int lpr = (hs4 % 8 == 0) ? 8 : (hs4 % 4 == 0) ? 4 : (hs4 % 2 == 0) ? 2 : 1;
    const int nf = hs4 / lpr;
    const int ng = NWARP * (32 / lpr);
    *smem = ((size_t)ng * head_size + 3 * (size_t)ng + 2 * (size_t)head_size + 4) * sizeof(float);
    switch (nf) {
    case 1: return attn_wo_kernel<1>;
    case 2: return attn_wo_kernel<2>;
    case 3: return attn_wo_kernel<3>;
    case 4: return attn_wo_kernel<4>;
    case 5: return attn_wo_kernel<5>;
    case 6: return attn_wo_kernel<6>;
    case 8: return attn_wo_kernel<8>;
    default: return nullptr;
    }
}

// attention + wo of one layer in one cluster launch (small models): partial vectors -> ctx->attn_parts
int launch_attn_wo(l2b_ctx *ctx, int layer, cudaStream_t st) {
    if (ctx->profiling) {
        const int hpos = ctx->n_appended > 0 ? ctx->n_appended - 1 : 0;
        int prc = prof_mark(ctx, "attn_wo", layer, 2ull * (uint64_t)(hpos + 1) * ctx->kv_loc * 4ull + (uint64_t)ctx->dim * ctx->q_loc * 4ull, st);
        if (prc) return prc;
    }
    AttnWoParams q{};
    AttnParams &a = q.a;
    a.ctl = ctx->ctl;
    a.q = ctx->q;
    const size_t loff = (size_t)layer * ctx->cfg.seq_len * ctx->kv_loc;   // :354
    a.kcache = ctx->kcache + loff;
    a.vcache = ctx->vcache + loff;
    a.head_size = ctx->head_size;
    a.kv_dim = ctx->kv_loc;
    a.kv_mul = ctx->kv_mul;
    a.trace = nullptr;
    q.wo = ctx->wo + (size_t)layer * ctx->dim * ctx->q_loc;
    q.parts = ctx->attn_parts;
    q.dim = ctx->dim;
    q.q_dim = ctx->q_loc;
    size_t smem = 0;
    attn_wo_fn fn = pick_attn_wo(ctx->head_size, &smem);
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(ctx->heads_loc, ctx->attn_R);
    lc.blockDim = dim3(NT);
    lc.dynamicSmemBytes = smem;
    lc.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = ctx->attn_R; at[0].val.clusterDim.z = 1;
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
        int prc = prof_mark(ctx, "attention", layer, 2ull * (uint64_t)(hpos + 1) * ctx->kv_loc * 4ull, st);
        if (prc) return prc;
    }
    AttnParams a{};
    a.ctl = ctx->ctl;
    a.q = q;
    const size_t loff = (size_t)layer * ctx->cfg.seq_len * ctx->kv_loc;   // :354
    a.kcache = ctx->kcache + loff;
    a.vcache = ctx->vcache + loff;
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
    a.trace = zb ? nullptr : trace_slot(ctx);
    const AttnBatch none{};
    size_t smem = ctx->attn_smem;
    attn_fn fn = pick_attention(ctx->head_size, ctx->attn_flash, &smem);
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(ctx->heads_loc, ctx->nsplit, nb);
    lc.blockDim = dim3(NT);
    lc.dynamicSmemBytes = smem;
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
    p.w0 = ctx->wq + (size_t)l * ctx->q_loc * dim;
    p.w1 = ctx->wk + (size_t)l * ctx->kv_loc * dim;
    p.w2 = ctx->wv + (size_t)l * ctx->kv_loc * dim;
    p.rows0 = ctx->q_loc; p.rows1 = ctx->kv_loc; p.rows2 = ctx->kv_loc;
    p.total_rows = ctx->q_loc + 2 * ctx->kv_loc;
    const size_t loff = (size_t)l * ctx->cfg.seq_len * ctx->kv_loc;
    p.kcache = ctx->kcache + loff;
    p.vcache = ctx->vcache + loff;
    p.rope_cos = ctx->rope_cos; p.rope_sin = ctx->rope_sin;
    p.head_size = ctx->head_size; p.kv_dim = ctx->kv_loc;
    // wo, whose result is added to the residual stream (:392-395)
    g.wo.ctl = ctx->ctl;
    g.wo.n = ctx->q_loc;
    g.wo.w0 = ctx->wo + (size_t)l * dim * ctx->q_loc;
    g.wo.total_rows = dim; g.wo.rows0 = dim;
    // rmsnorm + w1,w3 + SiLU*mul (:398-416)
    g.w13.ctl = ctx->ctl;
    g.w13.n = dim;
    g.w13.gamma = ctx->rms_ffn + (size_t)l * dim;
    g.w13.w0 = ctx->w1 + (size_t)l * ctx->hid_loc * dim;
    g.w13.w1 = ctx->w3 + (size_t)l * ctx->hid_loc * dim;
    g.w13.rows0 = ctx->hid_loc;
    g.w13.total_rows = 2 * ctx->hid_loc;
    // w2, added to the residual stream (:419-422)
    g.w2.ctl = ctx->ctl;
    g.w2.n = ctx->hid_loc;
    g.w2.w0 = ctx->w2 + (size_t)l * dim * ctx->hid_loc;
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
        for (int tpr : tprs) L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)gemv_pick(epi, tpr)));
        L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)gemv8_pick(epi)));
        L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)gemv_tma_pick(epi)));
    }
    size_t smem = 0;
    L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)pick_attention(ctx->head_size, true, &smem)));
    if (pick_attn_wo(ctx->head_size, &smem)) L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, (const void *)pick_attn_wo(ctx->head_size, &smem)));
    const void *others[] = {(const void *)attention_kernel, (const void *)advance_kernel,
                            (const void *)batch_advance_kernel, (const void *)gather_logits_kernel,
                            (const void *)resid_add_kernel, (const void *)sample_prep_kernel,
                            (const void *)sample_prep_batch_kernel, (const void *)logprob_kernel,
                            (const void *)logprob_batch_kernel, (const void *)synth_fill_kernel};
    for (const void *f : others) L2B_CUDA(ctx, cudaFuncGetAttributes(&fa, f));
    // The kernels that run next to a TMA-ring GEMV in a decode step (the ring GEMVs, attention, the
    // token advance) all ask for the largest shared-memory carveout, so consecutive kernels never
    // need a different L1 / shared split to share an SM: a ring kernel's successor enters while it drains.
    const void *decode[] = {(const void *)pick_attention(ctx->head_size, true, &smem), (const void *)attention_kernel,
                            (const void *)advance_kernel};
    for (const void *f : decode)
        L2B_CUDA(ctx, cudaFuncSetAttribute(f, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    for (int epi = 0; epi < EPI_COUNT; ++epi)
        L2B_CUDA(ctx, cudaFuncSetAttribute((const void *)gemv_tma_pick(epi), cudaFuncAttributePreferredSharedMemoryCarveout,
                                           cudaSharedmemCarveoutMaxShared));
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
    ctx->smem_per_sm = prop.sharedMemPerMultiprocessor;
    ctx->smem_reserved = prop.reservedSharedMemPerBlock;
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
    L2B_TRY(materialize(ctx, &ctx->emb, src, o_emb, 1, 1, V, dim, SH_NONE, {0.0, 0.04, -BIG, BIG}));
    L2B_TRY(materialize(ctx, &ctx->rms_att, src, o_ratt, 2, 1, L, dim, SH_NONE, {1.35, 0.35, 0.25f, 2.4f}));
    L2B_TRY(materialize(ctx, &ctx->wq, src, o_wq, 3, L, dim, dim, SH_ROWS, {0.0, 0.04 * sd, -BIG, BIG}));
    L2B_TRY(materialize(ctx, &ctx->wk, src, o_wk, 4, L, kvd, dim, SH_ROWS, {0.0, 0.04 * sd, -BIG, BIG}));
    L2B_TRY(materialize(ctx, &ctx->wv, src, o_wv, 5, L, kvd, dim, SH_ROWS, {0.0, 0.02 * sd, -BIG, BIG}));
    L2B_TRY(materialize(ctx, &ctx->wo, src, o_wo, 6, L, dim, dim, SH_COLS, {0.0, 0.02 * sd, -BIG, BIG}));
    L2B_TRY(materialize(ctx, &ctx->rms_ffn, src, o_rffn, 7, 1, L, dim, SH_NONE, {1.35, 0.35, 0.25f, 2.4f}));
    L2B_TRY(materialize(ctx, &ctx->w1, src, o_w1, 8, L, hid, dim, SH_ROWS, {0.0, 0.026 * sd, -BIG, BIG}));
    L2B_TRY(materialize(ctx, &ctx->w2, src, o_w2, 9, L, dim, hid, SH_COLS, {0.0, 0.026 * sh, -BIG, BIG}));
    L2B_TRY(materialize(ctx, &ctx->w3, src, o_w3, 10, L, hid, dim, SH_ROWS, {0.0, 0.026 * sd, -BIG, BIG}));
    L2B_TRY(materialize(ctx, &ctx->rms_final, src, o_rfin, 11, 1, 1, dim, SH_NONE, {7.1, 0.6, 3.0f, 10.0f}));
    if (cfg->shared_weights) {
        ctx->wcls = ctx->emb + (size_t)rank * ctx->vocab_loc * dim;   // :112
    } else {
        L2B_TRY(materialize(ctx, &ctx->wcls, src, o_wcls, 14, 1, V, dim, SH_ROWS, {0.0, 0.04, -BIG, BIG}));
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
    return create_run_state(ctx);
}

// run state, attention launch shape, pinned host buffers, tensor-parallel landing area and switches
// of one rank whose weights are in place
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
        size_t smem_aw = 0;
        ctx->fuse_attn = (want & 1) && world == 1 && dim < 1024 && pick_attn_wo((int)hs, &smem_aw) != nullptr;
        const char *er = getenv("L2B_ATTN_R");
        ctx->attn_R = er && atoi(er) >= 1 && atoi(er) <= 8 ? atoi(er) : 8;
        if (ctx->fuse_attn) L2B_TRY(dev_alloc(ctx, &ctx->attn_parts, (size_t)cfg->n_heads * dim));
    }
    L2B_TRY(dev_alloc(ctx, &ctx->delta, dim));
    L2B_TRY(dev_alloc(ctx, &ctx->q, (size_t)ctx->q_loc));
    L2B_TRY(dev_alloc(ctx, &ctx->xb, (size_t)ctx->q_loc));
    L2B_TRY(dev_alloc(ctx, &ctx->hb, (size_t)ctx->hid_loc));
    L2B_TRY(dev_alloc(ctx, &ctx->logits, V));
    if (world > 1) L2B_TRY(dev_alloc(ctx, &ctx->logits_loc, (size_t)ctx->vocab_loc));
    L2B_TRY(dev_alloc(ctx, &ctx->kcache, L * S * ctx->kv_loc));
    L2B_TRY(dev_alloc(ctx, &ctx->vcache, L * S * ctx->kv_loc));
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
    L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->kcache, 0, L * S * ctx->kv_loc * sizeof(float), ctx->stream), "memset"));
    L2B_TRY(cuda_try(ctx, cudaMemsetAsync(ctx->vcache, 0, L * S * ctx->kv_loc * sizeof(float), ctx->stream), "memset"));

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
        if (ctx->attn_smem > kMaxDynSmem) {
            ctx->err = "seq_len too large for the attention kernel's shared memory";
            g_create_error = ctx->err;
            return L2B_ERR_UNSUPPORTED;
        }
        L2B_TRY(cuda_try(ctx, cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem), "cudaFuncSetAttribute"));
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
        const char *envp = getenv("L2B_TPR_TILES");
        if (envp) ctx->tpr_min_tiles_per_sm = atoi(envp);
        const char *env6 = getenv("L2B_TMA_CTAS");
        if (env6) ctx->tma_ctas_per_sm = atoi(env6) > 0 ? atoi(env6) : 1;
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
    if (ctx->weights && --ctx->weights->refs == 0) {   // the last context or session of the model
        for (void *p : ctx->weights->owned) cudaFree(p);
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

int common_create(l2b_ctx **out, const l2b_config *cfg, const Source &src, uint64_t n_floats,
                  const float *rope_cos, const float *rope_sin, const l2b_shard *shard, int n_gpus) {
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
    if (in_process) ranks[0]->members = ranks;
    *out = ranks[0];
    return L2B_OK;
}

// a context on the weights of `model` (single GPU): its own run state, caches, stream and graphs
int create_session(l2b_ctx *ctx, const l2b_ctx *model) {
    L2B_TRY(init_rank(ctx, &model->cfg, 0, 1, model->device));
    ctx->weights = model->weights;
    ++ctx->weights->refs;
    ctx->emb = model->emb; ctx->rms_att = model->rms_att; ctx->rms_ffn = model->rms_ffn; ctx->rms_final = model->rms_final;
    ctx->wq = model->wq; ctx->wk = model->wk; ctx->wv = model->wv; ctx->wo = model->wo;
    ctx->w1 = model->w1; ctx->w2 = model->w2; ctx->w3 = model->w3; ctx->wcls = model->wcls;
    ctx->rope_cos = model->rope_cos; ctx->rope_sin = model->rope_sin;
    L2B_TRY(create_run_state(ctx));
    return warm_up(std::vector<l2b_ctx *>{ctx});
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

int finish_call(l2b_ctx *lead, const std::vector<l2b_ctx *> &ranks) {
    int rc = L2B_OK;
    for (l2b_ctx *c : ranks) {
        cudaSetDevice(c->device);
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
    int rc = L2B_OK;
    for (size_t i = 0; i < nranks; ++i) {
        l2b_ctx *c = ranks[i];
        if (nranks > 1) cudaSetDevice(c->device);
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
    if (rc) return rc;
    if (lead->time_steps) {
        if (nranks > 1) L2B_CUDA(lead, cudaSetDevice(lead->device));
        L2B_CUDA(lead, cudaEventElapsedTime(&lead->last_ms, lead->ev0, lead->ev1));
    }
    if (pos + 1 > lead->n_appended) lead->n_appended = pos + 1;
    return L2B_OK;
}

// The output of a sampling step, from ctx's pinned buffers: its probabilities to host_probs (if not
// NULL and not the pinned buffer itself), and with the candidate filter on its candidates and their
// count to cand / *n_cand, or minus their number when more passed than fit (the host then filters the
// probabilities itself).  Without the filter *n_cand = 0.
void copy_sample_out(l2b_ctx *ctx, bool filter, float *host_probs, l2b_prob_index *cand, int cand_cap, int32_t *n_cand) {
    const int V = ctx->cfg.vocab_size;
    if (host_probs && host_probs != ctx->h_logits) memcpy(host_probs, ctx->h_logits, (size_t)V * sizeof(float));
    if (n_cand) *n_cand = 0;
    if (filter) {
        const int n = ctx->h_ints[2];
        if (n > kCandCap || n > cand_cap) { *n_cand = -n; return; }   // too many: filter host_probs on the host
        static_assert(sizeof(l2b_prob_index) == sizeof(ProbIndex), "candidate layout");
        memcpy(cand, ctx->h_cand, (size_t)n * sizeof(ProbIndex));
        *n_cand = n;
    }
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
    copy_sample_out(ctx, filter, host_probs, cand, cand_cap, n_cand);
    return L2B_OK;
}

}  // extern "C" (templates below)

// ---- batched prompt prefill (prefill_gemm_kernel in l2b_device.cuh) -----------------------------
template <int NB>
gemv_fn pf_pick(int epi) {
    switch (epi) {
    case EPI_QKV: return prefill_gemm_kernel<EPI_QKV, NB>;
    case EPI_SILU: return prefill_gemm_kernel<EPI_SILU, NB>;
    case EPI_STORE: return prefill_gemm_kernel<EPI_STORE, NB>;
    case EPI_ARGMAX: return prefill_gemm_kernel<EPI_ARGMAX, NB>;
    default: return prefill_gemm_kernel<EPI_RESID, NB>;
    }
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
                           pick_attention(ctx->head_size, true, &smem) != attention_kernel &&
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
    if ((rc = dev_alloc(ctx, &ctx->pf_tokens, (size_t)ctx->cfg.seq_len))) return rc;
    L2B_CUDA(ctx, cudaMemsetAsync(ctx->pf_counters, 0, (size_t)PF_MAXB * ctx->heads_loc * sizeof(unsigned int), ctx->stream));
    for (int epi : {(int)EPI_QKV, (int)EPI_SILU, (int)EPI_RESID, (int)EPI_STORE, (int)EPI_ARGMAX}) {
        L2B_CUDA(ctx, cudaFuncSetAttribute(pf_pick<PF_MAXB>(epi), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPfSmemBudget));
        L2B_CUDA(ctx, cudaFuncSetAttribute(pf_pick<2>(epi), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPfSmemBudget));
    }
    ctx->pf_ok = true;
    return L2B_OK;
}

template <int NB>
static int pf_launch(l2b_ctx *ctx, int epi, GemvParams p, cudaStream_t st) {
    const size_t xbytes = (size_t)NB * p.n * 4;
    const int nstage = pf_ring_stages(kPfSmemBudget, xbytes);
    p.nstage = nstage;
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
    L2B_CUDA(ctx, cudaLaunchKernelEx(&lc, pf_pick<NB>(epi), p));
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
        const size_t loff = (size_t)l * ctx->cfg.seq_len * ctx->kv_loc;
        AttnBatch zb{};
        for (int b = 0; b < nb; ++b) {
            g.qkv.pos_b[b] = zb.pos[b] = pos[b];
            g.qkv.kcache_b[b] = kv[b]->kcache + loff;
            g.qkv.vcache_b[b] = kv[b]->vcache + loff;
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

// n_tokens positions starting at pos0, PF_MAXB per pass over the weights; KV cache filled.  Without
// score no logits; with score (l2b_score: tokens holds n_tokens + 1 entries) each group then runs the
// argmax classifier and logprob_batch_kernel, which leaves position i's log-probability of tokens[i + 1]
// and its greedy token in score_lp[i] and score_greedy[i].
static int prefill_batched(l2b_ctx *ctx, const int32_t *tokens, int n_tokens, int pos0, bool score = false) {
    cudaStream_t st = ctx->stream;
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    for (int i = 0; i < n_tokens; ++i) ctx->h_gen[i] = tokens[i];
    L2B_CUDA(ctx, cudaMemcpyAsync(ctx->pf_tokens, ctx->h_gen, (size_t)n_tokens * sizeof(int), cudaMemcpyHostToDevice, st));
    if (score) {   // the targets, from the caller's (pageable) array: staged before the call returns
        L2B_CUDA(ctx, cudaMemcpyAsync(ctx->gen_forced, tokens + 1, (size_t)n_tokens * sizeof(int), cudaMemcpyHostToDevice, st));
        L2B_CUDA(ctx, cudaMemsetAsync(ctx->pf_amax, 0, PF_MAXB * sizeof(unsigned long long), st));
    }
    fill_ctl(ctx, tokens[0], pos0, 0, 1.0f, -1.0f);          // DONE = 0 for the attention kernel
    L2B_CUDA(ctx, cudaMemcpyAsync(ctx->ctl, ctx->h_ctl, CTL_HOST_WORDS * sizeof(int), cudaMemcpyHostToDevice, st));
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev0, st));
    ctx->last_launches = 0;
    for (int done = 0; done < n_tokens; done += PF_MAXB) {
        const int nb = n_tokens - done < PF_MAXB ? n_tokens - done : PF_MAXB;
        l2b_ctx *kv[PF_MAXB];
        int pos[PF_MAXB];
        for (int b = 0; b < nb; ++b) { kv[b] = ctx; pos[b] = pos0 + done + b; }
        int rc = batched_layers(ctx, kv, pos, nb, ctx->pf_tokens + done, nullptr);
        if (rc) return rc;
        if (score) {
            rc = batched_classifier(ctx, nb, true);
            if (rc) return rc;
            rc = launch_logprob_batch(ctx, nb, done);
            if (rc) return rc;
        }
    }
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev1, st));
    L2B_CUDA(ctx, cudaStreamSynchronize(st));
    L2B_CUDA(ctx, cudaGetLastError());
    L2B_CUDA(ctx, cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
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
// score, their targets at gen_forced + done, their results to score_lp / score_greedy + done
static int launch_logprob_batch(l2b_ctx *ctx, int nb, int done) {
    LogprobBatchParams p{};
    p.ctl = ctx->ctl;
    p.logits = ctx->pf_logits;
    p.n = ctx->cfg.vocab_size;
    p.targets = ctx->gen_forced + done;
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

// sample_prep_batch_kernel over the nb logits rows of a group in pf_logits, in place; vector b is session
// s[b] (its candidates and count go to its own buffers) with temperature[b] and top_p[b] (< 0: no filter)
static int launch_sample_prep_batch(l2b_ctx *ctx, l2b_ctx *const *s, int nb, const float *temperature,
                                    const float *top_p) {
    SamplePrepBatchParams p{};
    p.ctl = ctx->ctl;
    p.logits = ctx->pf_logits;
    p.n = p.stride = ctx->cfg.vocab_size;
    p.cand_cap = kCandCap;
    for (int b = 0; b < nb; ++b) {
        p.temperature[b] = temperature[b];
        p.top_p[b] = top_p[b];
        p.cand[b] = s[b]->cand;
        p.n_cand[b] = s[b]->n_cand;
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
    int rc = pf_prepare(ctx);
    if (rc) return rc;
    // the vectors: vector v runs token tokens[v] at vpos[v] on session vs[v]; last[v]: the session it ends, or -1
    int total = 0;
    for (int i = 0; i < n; ++i) total += n_tok ? n_tok[i] : 1;
    std::vector<l2b_ctx *> vs(total);
    std::vector<int> vpos(total), last(total, -1);
    for (int i = 0, v = 0; i < n; ++i)
        for (int j = 0, len = n_tok ? n_tok[i] : 1; j < len; ++j, ++v) {
            vs[v] = s[i];
            vpos[v] = pos[i] + j;
            if (j == len - 1) last[v] = i;
        }
    cudaStream_t st = ctx->stream;
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->pf_ok) {
        // a run's leading tokens first, session by session; each prefill times itself on its session's events
        float pre_ms = 0.0f;
        int launches = 0;
        for (int v = 0, i = 0; v < total; ++v) {
            if (last[v] < 0) continue;
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
            const int i = last[v];
            if (i < 0) continue;
            rc = sample ? run_step(s[i], tokens[v], vpos[v], G_SAMPLE, temperature[i], top_p[i])
                        : run_step(s[i], tokens[v], vpos[v], argmax ? G_ARGMAX_ONE : G_LOGITS, 1.0f, 0.0f);
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
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev0, st));
    fill_ctl(ctx, tokens[0], pos[0], 0, 1.0f, -1.0f);        // DONE = 0 for the attention kernel
    L2B_CUDA(ctx, cudaMemcpyAsync(ctx->ctl, ctx->h_ctl, CTL_HOST_WORDS * sizeof(int), cudaMemcpyHostToDevice, st));
    ctx->last_launches = 0;
    for (int g = 0; g < total; g += PF_MAXB) {
        const int nb = total - g < PF_MAXB ? total - g : PF_MAXB;
        // from the caller's (pageable) array: staged before the call returns, ordered after the previous group
        L2B_CUDA(ctx, cudaMemcpyAsync(ctx->pf_tokens, tokens + g, (size_t)nb * sizeof(int), cudaMemcpyHostToDevice, st));
        rc = batched_layers(ctx, vs.data() + g, vpos.data() + g, nb, ctx->pf_tokens, nullptr);
        if (rc) return rc;
        // the group's vectors that end a run: row[k] in the group, of session ends[k]
        int row[PF_MAXB], nl = 0;
        l2b_ctx *ends[PF_MAXB];
        float lt[PF_MAXB], lp[PF_MAXB];
        for (int b = 0; b < nb; ++b) {
            const int i = last[g + b];
            if (i < 0) continue;
            row[nl] = b;
            ends[nl] = s[i];
            if (sample) { lt[nl] = temperature[i]; lp[nl] = top_p[i]; }
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
            rc = launch_sample_prep_batch(ctx, ends, nl, lt, lp);
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
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev1, st));
    L2B_CUDA(ctx, cudaStreamSynchronize(st));
    L2B_CUDA(ctx, cudaGetLastError());
    L2B_CUDA(ctx, cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
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
    int rc = finish_call(ctx, cs);
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
    int rc = pf_prepare(ctx);
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

static int forward_sample_runs(l2b_ctx *const *sessions, int32_t n, bool ragged, const int32_t *n_tok,
                               const int32_t *tokens, const int32_t *pos, const float *temperature,
                               const float *top_p, float *const *host_probs, l2b_prob_index *cand,
                               int32_t cand_cap, int32_t *n_cand) {
    int rc = check_batch_args(sessions, n, tokens, pos, ragged, n_tok);
    if (rc) return rc;
    l2b_ctx *s0 = sessions[0];
    if (!temperature || !top_p) return fail(s0, L2B_ERR_INVALID_ARG, "temperature or top_p is NULL");
    if (s0->cfg.vocab_size < 2) return fail(s0, L2B_ERR_INVALID_ARG, "sampling needs vocab_size >= 2");
    std::vector<float> filter_p(n);   // the kernel's top-p: < 0 = no filter
    for (int i = 0; i < n; ++i) {
        if (!(temperature[i] > 0.0f)) return fail(s0, L2B_ERR_INVALID_ARG, "temperature must be > 0 (use l2b_forward_argmax_batch for 0)");
        if (!(top_p[i] >= 0.0f && top_p[i] <= 1.0f)) return fail(s0, L2B_ERR_INVALID_ARG, "top_p must be in [0, 1]");
        const bool filter = (top_p[i] != 0.0f && top_p[i] != 1.0f);   // :1009
        if (filter && (!cand || !n_cand || cand_cap <= 0)) return fail(s0, L2B_ERR_INVALID_ARG, "candidate buffer missing");
        filter_p[i] = filter ? top_p[i] : -1.0f;
    }
    rc = step_sessions(sessions, n, ragged ? n_tok : nullptr, tokens, pos, MODE_SAMPLE, temperature, filter_p.data());
    if (rc) return rc;
    for (int i = 0; i < n; ++i)
        copy_sample_out(sessions[i], filter_p[i] >= 0.0f, host_probs ? host_probs[i] : nullptr,
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
    // the call's device ints: tokens, done flags, n_done, limits [n] each, the live count, then forced
    // and out_next [n][stride]
    const size_t o_tok = 0, o_done = (size_t)n, o_ndone = 2 * (size_t)n, o_lim = 3 * (size_t)n, o_live = 4 * (size_t)n;
    const size_t o_forced = o_live + 1, o_out = o_forced + (size_t)n * stride, total = o_out + (size_t)n * stride;
    L2B_CUDA(ctx, cudaSetDevice(ctx->device));
    if (ctx->gb_cap < total) {
        if (ctx->gb_ints) {
            L2B_CUDA(ctx, cudaFree(ctx->gb_ints));
            ctx->owned.erase(std::find(ctx->owned.begin(), ctx->owned.end(), (void *)ctx->gb_ints));
            ctx->gb_ints = nullptr;
            ctx->gb_cap = 0;
        }
        const int rc = dev_alloc(ctx, &ctx->gb_ints, total);
        if (rc) { cudaGetLastError(); return rc; }
        ctx->gb_cap = total;
    }
    std::vector<int> h(o_out, -1);
    for (int i = 0; i < n; ++i) {
        h[o_tok + i] = tokens[i];
        h[o_done + i] = 0;
        h[o_ndone + i] = 0;
        h[o_lim + i] = limit[i];
        if (forced)
            for (int k = 0; k < limit[i]; ++k) h[o_forced + (size_t)i * stride + k] = forced[(size_t)i * n_steps + k];
    }
    h[o_live] = n;
    int *d = ctx->gb_ints;
    cudaStream_t st = ctx->stream;
    L2B_CUDA(ctx, cudaMemcpyAsync(d, h.data(), o_out * sizeof(int), cudaMemcpyHostToDevice, st));
    L2B_CUDA(ctx, cudaMemsetAsync(ctx->pf_amax, 0, PF_MAXB * sizeof(unsigned long long), st));
    fill_ctl(ctx, tokens[0], pos[0], 0, 1.0f, -1.0f);        // DONE = 0 until the last session stops
    L2B_CUDA(ctx, cudaMemcpyAsync(ctx->ctl, ctx->h_ctl, CTL_HOST_WORDS * sizeof(int), cudaMemcpyHostToDevice, st));
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev0, st));
    ctx->last_launches = 0;
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
            int rc = batched_layers(ctx, s + g, p, nb, d + o_tok + g, d + o_done + g);
            if (rc) return rc;
            rc = batched_classifier(ctx, nb, true);
            if (rc) return rc;
            a.g0 = g; a.nb = nb; a.step = step;
            void *args[] = {&a};
            rc = launch_small(ctx, (const void *)batch_advance_kernel, dim3(1), dim3(PF_MAXB), args, st, true);
            if (rc) return rc;
        }
    }
    std::vector<int> back((size_t)n * stride + n);
    L2B_CUDA(ctx, cudaMemcpyAsync(back.data(), d + o_ndone, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
    L2B_CUDA(ctx, cudaMemcpyAsync(back.data() + n, d + o_out, (size_t)n * stride * sizeof(int), cudaMemcpyDeviceToHost, st));
    L2B_CUDA(ctx, cudaEventRecord(ctx->ev1, st));
    L2B_CUDA(ctx, cudaStreamSynchronize(st));
    L2B_CUDA(ctx, cudaGetLastError());
    L2B_CUDA(ctx, cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
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
    rc = pf_prepare(s0);
    if (rc) return rc;
    if (s0->pf_ok) return generate_batched(sessions, n, tokens, pos, n_steps, forced, limit.data(), stop_on_bos, out_next, n_done);
    return generate_each(sessions, n, tokens, pos, n_steps, forced, limit.data(), stop_on_bos, out_next, n_done);
}

int32_t l2b_read_state(l2b_ctx *ctx, int32_t which, float *dst, uint64_t n, uint64_t *n_out) {
    if (!ctx || !dst) return L2B_ERR_INVALID_ARG;
    const float *src = nullptr;
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
    L2B_CUDA(ctx, cudaMemcpy(dst, src, cnt * sizeof(float), cudaMemcpyDeviceToHost));
    if (n_out) *n_out = cnt;
    return L2B_OK;
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
        int r2 = finish_call(ctx, ranks);
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
    // SURVEY.md 8d: every weight touched once per token (+ the embedding row), this rank's shard
    uint64_t w = L * ((uint64_t)ctx->q_loc * dim + 2ull * ctx->kv_loc * dim + dim * ctx->q_loc +
                      3ull * ctx->hid_loc * dim + 2 * dim) +
                 dim + (uint64_t)ctx->vocab_loc * dim;
    if (weight_bytes) *weight_bytes = 4 * w;
    if (kv_bytes) *kv_bytes = 4ull * L * 2 * ctx->kv_loc * (uint64_t)(pos + 1);
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
    tmp.smem_per_sm = prop.sharedMemPerMultiprocessor;
    tmp.smem_reserved = prop.reservedSharedMemPerBlock;
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
    cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
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
