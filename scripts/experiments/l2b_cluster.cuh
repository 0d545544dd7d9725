// l2b_cluster.cuh — all layers of a small model's decode step in ONE thread-block-cluster kernel.
//
// stories15M-class models (dim <= 512) are latency-bound: a step is 31 dependent kernels of ~3 us
// that move 60 MB out of L2 (DESIGN.md 6).  What a kernel boundary costs there (completion, flush,
// dependency wait, TMA staging of x: ~2 us) a cluster barrier does in ~0.2 us (barrier.cluster +
// L1 flush) and a distributed-shared-memory gather in ~0.1 us.  So: one cluster of C CTAs (C = 16,
// non-portable size) runs every layer of the step; a layer is five phases separated by cluster
// barriers:
//   1  rmsnorm + this CTA's rows of [wq; wk; wv] + RoPE (:305-351); q slice stays in shared memory,
//      k / v rows go to the KV cache in global memory (:353-358)
//   2  attention (:361-389): CTA h handles head h — gathers q_h from the owners' shared memory,
//      flash-decoding over the cache, output xb_h stays in shared memory
//   3  gather xb; this CTA's rows of wo; x slice += (:392-395)
//   4  gather x; rmsnorm + this CTA's (w1, w3) row pairs + SiLU*mul (:398-416); hb slice
//   5  gather hb; this CTA's rows of w2; x slice += (:419-422)
// Results are exchanged by PULL: every CTA keeps the slice it produced in its own shared memory and
// the consumers read it through DSMEM after the barrier (a slice buffer is rewritten five barriers
// later, so no reader can still be on it).  The first weight tile of the NEXT phase is requested
// before each barrier, so its L2 round trip overlaps the barrier and the gather.
// Only 16 SMs work on the layers, so each phase is bound by those SMs' L2 ports; the classifier
// (60 % of the bytes) stays a separate full-chip kernel.
#pragma once

#include <cooperative_groups.h>

#include "l2b_device.cuh"

namespace l2b {

constexpr int CL_MAXU = 16;        // float4 columns per lane per row: n <= TPR * 16 * 4
constexpr int CL_MAX_C = 16;
__host__ __device__ __forceinline__ int cl_round4(int v) { return (v + 3) & ~3; }

struct ClusterParams {
    const float *emb, *rms_att, *rms_ffn;
    const float *wq, *wk, *wv, *wo, *w1, *w2, *w3;
    float *kcache, *vcache;             // (L, seq_len, kv_dim)
    const float *rope_cos, *rope_sin;   // (seq_len, head_size/2)
    int *ctl;
    float *x_out;                       // the residual stream after the last layer (input of the classifier kernel)
    int dim, hidden, n_layers, n_heads, kv_mul, head_size, kv_dim, seq_len;
    int bump_epoch;
    unsigned long long *trace;          // L2B_TRACE=1: [n_layers][32] phase stamps of CTA 0 (ns)
};

// one (row pair) x (TPR lanes) dot-product tile: weights of rows (v0, v0+1) in registers
template <int TPR, int U>
struct ClTile {
    float4 w[2][U];
};

// virtual-row pointers of the three GEMV flavours
__device__ __forceinline__ const float *cl_row_qkv(const ClusterParams &p, int l, int v) {
    const int qd = p.dim, kvd = p.kv_dim;
    if (v < qd) return p.wq + ((size_t)l * qd + v) * p.dim;
    v -= qd;
    if (v < kvd) return p.wk + ((size_t)l * kvd + v) * p.dim;
    v -= kvd;
    return p.wv + ((size_t)l * kvd + v) * p.dim;
}

// issue the loads of rows (v0, v0+1) [valid if < vend], n4 float4 columns, lane `sub` of TPR
template <int TPR, int U, class RowPtr>
__device__ __forceinline__ void cl_issue(ClTile<TPR, U> &t, RowPtr row_ptr, int v0, int vend, int n4, int sub) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const bool ok = v0 + r < vend;
        const float4 *wr = reinterpret_cast<const float4 *>(row_ptr(ok ? v0 + r : v0));
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int c = u * TPR + sub;
            t.w[r][u] = (ok && c < n4) ? ldg_stream(wr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
}

template <int TPR, int U>
__device__ __forceinline__ void cl_dot(const ClTile<TPR, U> &t, const float4 *xs4, int n4, int sub, float &a0, float &a1) {
    a0 = 0.0f; a1 = 0.0f;
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const int c = u * TPR + sub;
        if (c < n4) {
            const float4 xv = xs4[c];
            a0 = dot4(t.w[0][u], xv, a0);
            a1 = dot4(t.w[1][u], xv, a1);
        }
    }
#pragma unroll
    for (int o = (TPR < 32 ? TPR : 32) / 2; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
}

// rmsnorm of src (n <= 2 * NT floats, shared memory) into dst (shared memory); the gain of elements
// tid and tid + NT is already in registers (fetched a phase earlier: its L2 round trip is hidden)
__device__ __forceinline__ void cl_rmsnorm(float *dst, const float *src, const float (&g)[2], int n, float *scratch) {
    const int tid = threadIdx.x;
    const float v0 = tid < n ? src[tid] : 0.0f, v1 = tid + NT < n ? src[tid + NT] : 0.0f;
    float ssq = fmaf(v0, v0, 0.0f);
    ssq = fmaf(v1, v1, ssq);
    float ss = block_sum(ssq, scratch);
    ss /= (float)n;            // :452
    ss += 1e-5f;               // :453
    const float s = 1.0f / sqrtf(ss);   // :454
    if (tid < n) dst[tid] = __fmul_rn(__fmul_rn(v0, s), g[0]);            // :462
    if (tid + NT < n) dst[tid + NT] = __fmul_rn(__fmul_rn(v1, s), g[1]);
    __syncthreads();
}
__device__ __forceinline__ void cl_load_gain(float (&g)[2], const float *gamma, int n) {
    const int tid = threadIdx.x;
    g[0] = tid < n ? __ldg(gamma + tid) : 0.0f;
    g[1] = tid + NT < n ? __ldg(gamma + tid + NT) : 0.0f;
}

// NF: attention float4 per lane per row (head_size = 4 * NF * LPR); U8 >= ceil(dim/4/8) and
// U16 >= ceil(hidden/4/16): float4 columns per lane of the two GEMV tile shapes (register arrays)
template <int NF, int U8, int U16>
__global__ void __launch_bounds__(NT, 1) layers_cluster_kernel(const ClusterParams p) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int C = gridDim.x, rank = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dim = p.dim, hidden = p.hidden, hs = p.head_size, hs4 = hs >> 2;
    const int n4 = dim >> 2;
    const int qkv_rows = dim + 2 * p.kv_dim;
    // per-CTA slices (even row counts so that RoPE / (w1,w3) pairs never straddle two CTAs)
    auto slice = [&](int rows, int &r0, int &r1) {
        int per = (rows + C - 1) / C;
        per += per & 1;
        r0 = min(rows, rank * per);
        r1 = min(rows, r0 + per);
        return per;
    };
    int q0, q1, x0, x1, h0, h1;
    const int qkv_per = slice(qkv_rows, q0, q1);
    const int x_per = slice(dim, x0, x1);
    const int hb_per = slice(hidden, h0, h1);      // hidden units; virtual rows are 2x

    // ---- shared memory carve-up
    float *xres = reinterpret_cast<float *>(smem_raw);        // [dim]      residual stream (full copy)
    float *vin = xres + dim;                                  // [max(dim, hidden)] GEMV input
    const int vmax = dim > hidden ? dim : hidden;
    const int hpc = (p.n_heads + C - 1) / C;                  // heads per CTA
    float *o_qkv = vin + vmax;                                // [qkv_per]  my rows of (q | k | v) after RoPE
    float *o_xb = o_qkv + cl_round4(qkv_per);                 // [hpc][hs]  attention output of my head(s)
    float *o_x = o_xb + hpc * hs;                             // [x_per]    my slice of the new x
    float *o_hb = o_x + cl_round4(x_per);                     // [hb_per]   my slice of hb
    float *att = o_hb + cl_round4(hb_per);                    // attention scratch: [NG][hs] + 3 NG (+pad) + hs
    __shared__ float scratch[NWARP + 1];
    __shared__ float sh_L, sh_M;

    const int LPR = hs4 / NF, RPW = 32 / LPR, NG = NWARP * RPW;
    float *accp = att, *mlp = accp + (size_t)NG * hs, *wgt = mlp + 2 * NG, *qh = wgt + cl_round4(NG);

    // ---- everything immutable that layer 0 needs is requested before the dependency wait
    ClTile<8, U8> t8, t8b;
    const int grp8 = tid >> 3, sub8 = tid & 7;               // TPR = 8: 32 row pairs (64 rows) per tile
    const int grp16 = tid >> 4, sub16 = tid & 15;            // TPR = 16: 16 row pairs (32 rows) per tile
    const int hid4 = hidden >> 2;
    cl_issue<8, U8>(t8, [&](int v) { return cl_row_qkv(p, 0, v); }, q0 + 2 * grp8, q1, n4, sub8);
    float g_att[2], g_ffn[2];
    cl_load_gain(g_att, p.rms_att, dim);
    cl_load_gain(g_ffn, p.rms_ffn, dim);

    // gather plans (the same every layer): which peer's slice holds the float2 this thread fetches
    constexpr int GX = 1, GH = 4;                             // dim <= 512 -> <= 256 pairs; hidden <= 2048 -> <= 1024 pairs
    const float2 *gx_src[GX], *gxb_src[GX], *gh_src[GH];
#pragma unroll
    for (int k = 0; k < GX; ++k) {
        const int e = 2 * (tid + k * NT);
        gx_src[k] = gxb_src[k] = nullptr;
        if (e < dim) {
            const int ox = e / x_per;
            gx_src[k] = reinterpret_cast<const float2 *>(cluster.map_shared_rank(o_x, ox) + (e - ox * x_per));
            const int h = e / hs;
            gxb_src[k] = reinterpret_cast<const float2 *>(cluster.map_shared_rank(o_xb, h % C) + ((h / C) * hs + e - h * hs));
        }
    }
#pragma unroll
    for (int k = 0; k < GH; ++k) {
        const int e = 2 * (tid + k * NT);
        gh_src[k] = nullptr;
        if (e < hidden) {
            const int oh = e / hb_per;
            gh_src[k] = reinterpret_cast<const float2 *>(cluster.map_shared_rank(o_hb, oh) + (e - oh * hb_per));
        }
    }
    auto gather_x = [&]() {
#pragma unroll
        for (int k = 0; k < GX; ++k)
            if (gx_src[k]) reinterpret_cast<float2 *>(xres)[tid + k * NT] = *gx_src[k];
        __syncthreads();
    };

    pdl_launch_dependents();
    pdl_wait();
    if (p.ctl[CTL_DONE]) return;                              // uniform over the cluster
    const int token = p.ctl[CTL_TOKEN], pos = p.ctl[CTL_POS];
    if (p.bump_epoch && rank == 0 && tid == 0) p.ctl[CTL_EPOCH] += 1;
    const int T = pos + 1;
    const float root_hs = sqrtf((float)hs);

    // RoPE factors of the row pair this thread finishes in the first q/k/v tile: the same rows every layer
    float rope_c = 1.0f, rope_s = 0.0f;
    {
        const int v = q0 + 2 * grp8;
        if (sub8 == 0 && v < q1 && v < dim + p.kv_dim) {
            const int i = v < dim ? v : v - dim;
            const int pr = (i % hs) >> 1;
            rope_c = __ldg(p.rope_cos + (size_t)pos * (hs >> 1) + pr);
            rope_s = __ldg(p.rope_sin + (size_t)pos * (hs >> 1) + pr);
        }
    }
    for (int i = tid; i < dim; i += NT) xres[i] = __ldg(p.emb + (size_t)token * dim + i);   // :295-296
    __syncthreads();

    // attention lanes
    const int LPRc = LPR;
    const int lr = lane % LPRc, rw = lane / LPRc, agrp = warp * RPW + rw;

#define CL_STAMP(k) do { if (p.trace && rank == 0 && tid == 0) p.trace[l * 32 + (k)] = global_ns(); } while (0)
    for (int l = 0; l < p.n_layers; ++l) {
        const size_t loff = (size_t)l * p.seq_len * p.kv_dim;
        CL_STAMP(0);
        // =========== phase 1: rmsnorm + q,k,v rows + RoPE + KV append (:305-358)
        cl_rmsnorm(vin, xres, g_att, dim, scratch);
        CL_STAMP(16);
        for (int v0 = q0; v0 < q1; v0 += 64) {               // 32 row pairs per tile
            const int v = v0 + 2 * grp8;
            if (v0 != q0) cl_issue<8, U8>(t8, [&](int vv) { return cl_row_qkv(p, l, vv); }, v, q1, n4, sub8);
            float a0, a1;
            cl_dot<8, U8>(t8, reinterpret_cast<const float4 *>(vin), n4, sub8, a0, a1);
            if (sub8 == 0 && v < q1) {
                if (v < dim + p.kv_dim) {                     // q or k: rotate the adjacent pair (:336-351)
                    const bool is_q = v < dim;
                    const int i = is_q ? v : v - dim;
                    float fcr = rope_c, fci = rope_s;
                    if (v0 != q0) {
                        const int pr = (i % hs) >> 1;
                        fcr = __ldg(p.rope_cos + (size_t)pos * (hs >> 1) + pr);
                        fci = __ldg(p.rope_sin + (size_t)pos * (hs >> 1) + pr);
                    }
                    const float r0v = __fsub_rn(__fmul_rn(a0, fcr), __fmul_rn(a1, fci));     // :348
                    const float r1v = __fadd_rn(__fmul_rn(a0, fci), __fmul_rn(a1, fcr));     // :349
                    if (is_q) { o_qkv[v - q0] = r0v; o_qkv[v - q0 + 1] = r1v; }
                    else *reinterpret_cast<float2 *>(p.kcache + loff + (size_t)pos * p.kv_dim + i) = make_float2(r0v, r1v);   // :355
                } else {
                    const int i = v - dim - p.kv_dim;
                    *reinterpret_cast<float2 *>(p.vcache + loff + (size_t)pos * p.kv_dim + i) = make_float2(a0, a1);          // :356
                }
            }
        }
        CL_STAMP(17);
        // requested before the barrier: my first wo tile, and (attention CTAs) the cache rows of the
        // earlier positions for my head's first pass - only the row of `pos` itself is new
        cl_issue<8, U8>(t8b, [&](int v) { return p.wo + ((size_t)l * dim + v) * dim; }, x0 + 2 * grp8, x1, n4, sub8);
        float4 kk0[NF], vv0[NF];
        const bool pre_ok = rank < p.n_heads && agrp < pos;   // row t = agrp of head `rank`, already in the cache
        if (pre_ok) {
            const size_t hoff0 = (size_t)(rank / p.kv_mul) * hs;
            const float4 *k4 = reinterpret_cast<const float4 *>(p.kcache + loff + hoff0 + (size_t)agrp * p.kv_dim);
            const float4 *v4 = reinterpret_cast<const float4 *>(p.vcache + loff + hoff0 + (size_t)agrp * p.kv_dim);
#pragma unroll
            for (int f = 0; f < NF; ++f) { kk0[f] = __ldcg(k4 + lr + f * LPRc); vv0[f] = __ldcg(v4 + lr + f * LPRc); }
        }
        CL_STAMP(18);
        __threadfence();                                      // k / v rows visible to the attention CTAs
        CL_STAMP(1);
        cluster.sync();
        CL_STAMP(2);

        // =========== phase 2: attention, head h on CTA h (:361-389)
        for (int h = rank; h < p.n_heads; h += C) {
            // gather q_h from the owners of rows h*hs .. (h+1)*hs
            if (tid < hs) {
                const int v = h * hs + tid;
                const int owner = v / qkv_per;
                qh[tid] = cluster.map_shared_rank(o_qkv, owner)[v - owner * qkv_per];
            }
            __syncthreads();
            CL_STAMP(19);
            const float4 *q4 = reinterpret_cast<const float4 *>(qh);
            const size_t hoff = (size_t)(h / p.kv_mul) * hs;
            const float *kb = p.kcache + loff + hoff, *vb = p.vcache + loff + hoff;
            float4 qf[NF], acc[NF];
#pragma unroll
            for (int f = 0; f < NF; ++f) { qf[f] = q4[lr + f * LPRc]; acc[f] = make_float4(0.f, 0.f, 0.f, 0.f); }
            float m = -INFINITY, lsum = 0.0f;
            for (int tb = warp * RPW; tb < T; tb += NG) {     // warp-uniform bound
                const int t = tb + rw;
                const bool valid = t < T;
                float4 kk[NF], vv[NF];
                if (h == rank && tb == warp * RPW && pre_ok) {
#pragma unroll
                    for (int f = 0; f < NF; ++f) { kk[f] = kk0[f]; vv[f] = vv0[f]; }
                } else {
                    const float4 *k4 = reinterpret_cast<const float4 *>(kb + (size_t)(valid ? t : 0) * p.kv_dim);
                    const float4 *v4 = reinterpret_cast<const float4 *>(vb + (size_t)(valid ? t : 0) * p.kv_dim);
#pragma unroll
                    for (int f = 0; f < NF; ++f) { kk[f] = __ldcg(k4 + lr + f * LPRc); vv[f] = __ldcg(v4 + lr + f * LPRc); }
                }
                float sc = 0.0f;
#pragma unroll
                for (int f = 0; f < NF; ++f) sc = dot4(kk[f], qf[f], sc);
                for (int o = LPRc >> 1; o > 0; o >>= 1) sc += __shfl_xor_sync(0xffffffffu, sc, o);
                if (valid) {
                    sc = sc / root_hs;                        // :372
                    const float mn = fmaxf(m, sc);
                    const float scale = expf(m - mn), pw = expf(sc - mn);
                    lsum = fmaf(lsum, scale, pw);
#pragma unroll
                    for (int f = 0; f < NF; ++f) {
                        acc[f].x = fmaf(acc[f].x, scale, pw * vv[f].x);
                        acc[f].y = fmaf(acc[f].y, scale, pw * vv[f].y);
                        acc[f].z = fmaf(acc[f].z, scale, pw * vv[f].z);
                        acc[f].w = fmaf(acc[f].w, scale, pw * vv[f].w);
                    }
                    m = mn;
                }
            }
            CL_STAMP(20);
#pragma unroll
            for (int f = 0; f < NF; ++f) reinterpret_cast<float4 *>(accp + (size_t)agrp * hs)[lr + f * LPRc] = acc[f];
            if (lr == 0) { mlp[2 * agrp] = m; mlp[2 * agrp + 1] = lsum; }
            __syncthreads();
            if (warp == 0) {
                float M = -INFINITY;
                for (int g = lane; g < NG; g += 32) M = fmaxf(M, mlp[2 * g]);
                M = warp_max(M);
                float L = 0.0f;
                for (int g = lane; g < NG; g += 32) {
                    const float w = (mlp[2 * g] == -INFINITY) ? 0.0f : expf(mlp[2 * g] - M);
                    wgt[g] = w;
                    L = fmaf(w, mlp[2 * g + 1], L);
                }
                L = warp_sum(L);
                if (lane == 0) { sh_L = L; sh_M = M; }
            }
            __syncthreads();
            CL_STAMP(21);
            if (tid < hs) {
                float o = 0.0f;
                for (int g = 0; g < NG; ++g) o = fmaf(wgt[g], accp[(size_t)g * hs + tid], o);
                o_xb[(h / C) * hs + tid] = o / sh_L;          // :703-705
            }
            __syncthreads();
        }
        CL_STAMP(3);
        cluster.sync();
        CL_STAMP(4);

        // =========== phase 3: gather xb; my rows of wo; x slice += (:392-395)
#pragma unroll
        for (int k = 0; k < GX; ++k)
            if (gxb_src[k]) reinterpret_cast<float2 *>(vin)[tid + k * NT] = *gxb_src[k];
        __syncthreads();
        for (int v0 = x0; v0 < x1; v0 += 64) {
            const int v = v0 + 2 * grp8;
            if (v0 != x0) cl_issue<8, U8>(t8b, [&](int vv) { return p.wo + ((size_t)l * dim + vv) * dim; }, v, x1, n4, sub8);
            float a0, a1;
            cl_dot<8, U8>(t8b, reinterpret_cast<const float4 *>(vin), n4, sub8, a0, a1);
            if (sub8 == 0 && v < x1) {
                o_x[v - x0] = xres[v] + a0;                   // accum(), :708-713
                if (v + 1 < x1) o_x[v - x0 + 1] = xres[v + 1] + a1;
            }
        }
        // the first TWO (w1, w3) tiles for phase 4 (stories15M: 96 virtual rows per CTA = 1.5 tiles)
        auto w13_row = [&](int vv) { return ((vv & 1) ? p.w3 : p.w1) + ((size_t)l * hidden + (vv >> 1)) * dim; };
        cl_issue<8, U8>(t8, w13_row, 2 * h0 + 2 * grp8, 2 * h1, n4, sub8);
        cl_issue<8, U8>(t8b, w13_row, 2 * h0 + 64 + 2 * grp8, 2 * h1, n4, sub8);
        CL_STAMP(5);
        cluster.sync();
        CL_STAMP(6);
        gather_x();
        CL_STAMP(7);

        // =========== phase 4: rmsnorm + (w1, w3) row pairs + SiLU*mul (:398-416)
        cl_rmsnorm(vin, xres, g_ffn, dim, scratch);
        CL_STAMP(22);
        for (int v0 = 2 * h0, k = 0; v0 < 2 * h1; v0 += 64, ++k) {
            const int v = v0 + 2 * grp8;
            if (k >= 2) cl_issue<8, U8>(t8, w13_row, v, 2 * h1, n4, sub8);
            float a0, a1;
            if (k == 1) cl_dot<8, U8>(t8b, reinterpret_cast<const float4 *>(vin), n4, sub8, a0, a1);
            else cl_dot<8, U8>(t8, reinterpret_cast<const float4 *>(vin), n4, sub8, a0, a1);
            if (sub8 == 0 && v < 2 * h1) {
                const float sg = __fmul_rn(a0, __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-a0))));   // :412
                o_hb[(v >> 1) - h0] = __fmul_rn(sg, a1);                                      // :416
            }
        }
        CL_STAMP(23);
        // first w2 tile for phase 5: 16 lanes per row pair over the hidden columns, 32 rows per tile;
        // and the gains of the next layer
        ClTile<16, U16> t16;
        cl_issue<16, U16>(t16, [&](int v) { return p.w2 + ((size_t)l * dim + v) * hidden; }, x0 + 2 * grp16, x1, hid4, sub16);
        if (l + 1 < p.n_layers) {
            cl_load_gain(g_att, p.rms_att + (size_t)(l + 1) * dim, dim);
            cl_load_gain(g_ffn, p.rms_ffn + (size_t)(l + 1) * dim, dim);
        }
        CL_STAMP(8);
        cluster.sync();
        CL_STAMP(9);

        // =========== phase 5: gather hb; my rows of w2; x slice += (:419-422)
#pragma unroll
        for (int k = 0; k < GH; ++k)
            if (gh_src[k]) reinterpret_cast<float2 *>(vin)[tid + k * NT] = *gh_src[k];
        __syncthreads();
        for (int v0 = x0; v0 < x1; v0 += 32) {
            const int v = v0 + 2 * grp16;
            if (v0 != x0) cl_issue<16, U16>(t16, [&](int vv) { return p.w2 + ((size_t)l * dim + vv) * hidden; }, v, x1, hid4, sub16);
            float a0, a1;
            cl_dot<16, U16>(t16, reinterpret_cast<const float4 *>(vin), hid4, sub16, a0, a1);
            if (sub16 == 0 && v < x1) {
                o_x[v - x0] = xres[v] + a0;
                if (v + 1 < x1) o_x[v - x0 + 1] = xres[v + 1] + a1;
            }
        }
        // first q/k/v tile of the next layer
        if (l + 1 < p.n_layers)
            cl_issue<8, U8>(t8, [&](int v) { return cl_row_qkv(p, l + 1, v); }, q0 + 2 * grp8, q1, n4, sub8);
        CL_STAMP(10);
        cluster.sync();
        CL_STAMP(11);
        gather_x();
        CL_STAMP(12);
    }
#undef CL_STAMP
    if (rank == 0)
        for (int i = tid; i < dim; i += NT) p.x_out[i] = xres[i];
    cluster.sync();          // nobody leaves while a peer may still read its shared memory
}

}  // namespace l2b
