// Parked experiment (round 2): rmsnorm + w1/w3 + SiLU + the matching column slice of w2 per 32 hidden units in
// one kernel.  Parity-green; not part of the build and not measured on H100.  Was part of csrc/l2b_device.cuh; needs GemvParams / gemv_stage_input from there.
constexpr int FFN_HSZ = 32;       // hidden units per CTA = NT / 8 (one (w1, w3) row pair per 8-lane group)
constexpr int FFN_MAXU = 16;      // float4 columns per lane: dim <= 8 * 16 * 4 = 512
struct FfnParams {
    GemvParams g;           // prologue: x_in, parts/nparts, gamma, x_out, n = dim, ctl
    const float *w1, *w3;   // this layer's (hidden, dim)
    const float *w2;        // this layer's (dim, hidden)
    float *out_parts;       // (hidden / 32, dim)
    int hidden;
};

__global__ void __launch_bounds__(NT) ffn_fused_kernel(const FfnParams q) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const GemvParams &p = q.g;
    float *xs = reinterpret_cast<float *>(smem_raw);   // dim floats
    float *aux = xs + p.n;                              // gamma (dim) then the parts sum (dim)
    __shared__ uint64_t bar;
    __shared__ float scratch[NWARP + 1];
    __shared__ __align__(16) float hb_s[FFN_HSZ];
    const int tid = threadIdx.x, grp = tid >> 3, sub = tid & 7;
    const int n4 = p.n >> 2;
    const int j = blockIdx.x;                           // hidden slice [j*32, j*32+32)
    const int hrow = j * FFN_HSZ + grp;

    // ---- immutable weights first: this lane's share of one (w1, w3) row pair, and of the first w2 pass
    float4 wa[FFN_MAXU], wb[FFN_MAXU];
    {
        const float4 *r1 = reinterpret_cast<const float4 *>(q.w1 + (size_t)hrow * p.n);
        const float4 *r3 = reinterpret_cast<const float4 *>(q.w3 + (size_t)hrow * p.n);
#pragma unroll
        for (int u = 0; u < FFN_MAXU; ++u) {
            const int c = u * 8 + sub;
            wa[u] = (c < n4) ? ldg_stream(r1 + c) : make_float4(0.f, 0.f, 0.f, 0.f);
            wb[u] = (c < n4) ? ldg_stream(r3 + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    if (tid == 0) {
        mbar_init(&bar, 1);
        mbar_fence_init();
    }
    pdl_launch_dependents();
    pdl_wait();
    if (p.ctl[CTL_DONE]) return;
    gemv_stage_input(p, xs, aux, &bar, scratch);

    // ---- hb slice = silu(w1 . xs) * (w3 . xs)
    const float4 *xs4 = reinterpret_cast<const float4 *>(xs);
    float a0 = 0.0f, a1 = 0.0f;
#pragma unroll
    for (int u = 0; u < FFN_MAXU; ++u) {
        const int c = u * 8 + sub;
        if (c < n4) {
            const float4 xv = xs4[c];
            a0 = dot4(wa[u], xv, a0);
            a1 = dot4(wb[u], xv, a1);
        }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    if (sub == 0) {
        const float sg = __fmul_rn(a0, __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-a0))));   // :412
        hb_s[grp] = __fmul_rn(sg, a1);                                                // :416
    }
    __syncthreads();

    // ---- partial of w2: out[i] = sum_{k in slice} w2[i][j*32 + k] * hb[k]; 2 lanes per row, 4 float4 each
    const float4 *hb4 = reinterpret_cast<const float4 *>(hb_s);
    const int half = tid & 1;
    const float4 *w24 = reinterpret_cast<const float4 *>(q.w2) + (size_t)j * (FFN_HSZ / 4) + half * 4;
    const int h4 = q.hidden >> 2;
    for (int ib = 0; ib < p.n; ib += NT / 2) {           // warp-uniform bound
        const int i = ib + (tid >> 1);
        const bool valid = i < p.n;
        float a = 0.0f;
#pragma unroll
        for (int f = 0; f < 4; ++f) {
            const float4 w = valid ? ldg_stream(w24 + (size_t)i * h4 + f) : make_float4(0.f, 0.f, 0.f, 0.f);
            a = dot4(w, hb4[half * 4 + f], a);
        }
        a += __shfl_xor_sync(0xffffffffu, a, 1);
        if (valid && half == 0) q.out_parts[(size_t)j * p.n + i] = a;
    }
}

