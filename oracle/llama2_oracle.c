/*
 * llama2_oracle.c — CPU parity oracle (TEST INFRASTRUCTURE, see llama2_oracle.h).
 * Restates src/main.zig:285-713 plus the checkpoint layout
 * (:73-115, :936-967) and the temperature-0 generation loop (:995-1042).
 */
#define _POSIX_C_SOURCE 200809L
#include "llama2_oracle.h"

#include <math.h>
#include <pthread.h>
#include <unistd.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#ifndef ORC_OPTIMIZED
#define ORC_OPTIMIZED 0
#endif

#define ORC_W 4
#include "orc_simd_body.inc"
#undef ORC_W
#define ORC_W 8
#include "orc_simd_body.inc"
#undef ORC_W
#define ORC_W 16
#include "orc_simd_body.inc"
#undef ORC_W

#define ORC_DISPATCH(W, call)                   \
    do {                                        \
        if ((W) == 4) { call(_w4); }            \
        else if ((W) == 16) { call(_w16); }     \
        else { call(_w8); }                     \
    } while (0)

/* ---- primitive ops --------------------------------------------------------- */
void orc_matmul(float *xout, const float *x, const float *w, int d, int n, int W) {
    float *outs[1] = {xout};
    const float *ws[1] = {w};
#define CALL(sfx) matmul_fused##sfx(1, outs, x, ws, d, n)
    ORC_DISPATCH(W, CALL);
#undef CALL
}
void orc_matmul_fused2(float *o0, float *o1, const float *x, const float *w0, const float *w1,
                       int d, int n, int W) {
    float *outs[2] = {o0, o1};
    const float *ws[2] = {w0, w1};
#define CALL(sfx) matmul_fused##sfx(2, outs, x, ws, d, n)
    ORC_DISPATCH(W, CALL);
#undef CALL
}
void orc_matmul_fused3(float *o0, float *o1, float *o2, const float *x, const float *w0,
                       const float *w1, const float *w2, int d, int n, int W) {
    float *outs[3] = {o0, o1, o2};
    const float *ws[3] = {w0, w1, w2};
#define CALL(sfx) matmul_fused##sfx(3, outs, x, ws, d, n)
    ORC_DISPATCH(W, CALL);
#undef CALL
}
void orc_rmsnorm(float *o, const float *x, const float *w, int n, int W) {
#define CALL(sfx) rmsnorm##sfx(o, x, w, n)
    ORC_DISPATCH(W, CALL);
#undef CALL
}
float orc_dot(const float *x, const float *y, int n, int W) {
    float r;
#define CALL(sfx) r = dot##sfx(x, y, n)
    ORC_DISPATCH(W, CALL);
#undef CALL
    return r;
}
void orc_vector_mul(float *x, const float *y, int n, int W) {
#define CALL(sfx) vector_mul##sfx(x, y, n)
    ORC_DISPATCH(W, CALL);
#undef CALL
}
void orc_weighted_sum_rows(float *xout, int out_len, const float *rows, int row_stride,
                           const float *weights, int n_weights, int W) {
#define CALL(sfx) weighted_sum_rows##sfx(xout, out_len, rows, row_stride, weights, n_weights)
    ORC_DISPATCH(W, CALL);
#undef CALL
}

/* softmax, src/main.zig:687-706: scalar and sequential on purpose. */
void orc_softmax(float *x, int n) {
    float max = x[0];
    for (int i = 1; i < n; ++i)
        if (x[i] > max) max = x[i];
    float sum = 0.0f;
    for (int i = 0; i < n; ++i) {
        x[i] = expf(x[i] - max);
        sum += x[i];
    }
    for (int i = 0; i < n; ++i) x[i] /= sum;
}

/* accum, src/main.zig:708-713. */
void orc_accum(float *a, const float *b, int n) {
    for (int i = 0; i < n; ++i) a[i] += b[i];
}

/* argmax, src/main.zig:715-726. */
int orc_argmax(const float *x, int n) {
    float max = x[0];
    int maxi = 0;
    for (int i = 1; i < n; ++i)
        if (x[i] > max) {
            max = x[i];
            maxi = i;
        }
    return maxi;
}

/* RoPE angle, src/main.zig:338-342: freq = 1/pow(10000, (i % hs)/hs); val = pos*freq. */
void orc_rope_angle(int i, int head_size, int pos, float *fcr, float *fci) {
    const float head_dim = (float)(i % head_size);
    const float freq = 1.0f / powf(10000.0f, head_dim / (float)head_size);
    const float val = (float)pos * freq;
    *fcr = cosf(val);
    *fci = sinf(val);
}

/* ---- model ----------------------------------------------------------------- */
struct orc_model {
    orc_config cfg;
    int W;
    /* Weights, src/main.zig:53-71 */
    const float *token_embedding_table, *rms_att_weight, *rms_ffn_weight, *wq, *wk, *wv, *wo,
        *w1, *w2, *w3, *rms_final_weight, *freq_cis_real, *freq_cis_imag, *wcls;
    /* RunState, src/main.zig:119-135 */
    float *x, *xb, *xb2, *hb, *hb2, *q, *k, *v, *att, *logits, *key_cache, *value_cache;
};

uint64_t orc_checkpoint_floats(const orc_config *c, int shared_weights) {
    const uint64_t dim = c->dim, hid = c->hidden_dim, L = c->n_layers, V = c->vocab_size,
                   S = c->seq_len;
    const uint64_t hs = dim / c->n_heads, kvd = hs * c->n_kv_heads;
    uint64_t n = V * dim + L * dim + L * dim * dim + 2 * L * dim * kvd + L * dim * dim + L * dim +
                 3 * L * dim * hid + dim + 2 * (S * hs / 2);
    if (!shared_weights) n += V * dim;
    return n;
}

static float *orc_alloc(uint64_t n) {
    void *p = NULL;
    if (posix_memalign(&p, 64, (n ? n : 1) * sizeof(float)) != 0) return NULL;
    memset(p, 0, (n ? n : 1) * sizeof(float));
    return (float *)p;
}

orc_model *orc_model_create(const orc_config *c, const float *data, int shared_weights, int W) {
    if (W != 4 && W != 8 && W != 16) return NULL;
    orc_model *m = (orc_model *)calloc(1, sizeof(orc_model));
    if (!m) return NULL;
    m->cfg = *c;
    m->W = W;
    const uint64_t dim = c->dim, hid = c->hidden_dim, L = c->n_layers, V = c->vocab_size,
                   S = c->seq_len, H = c->n_heads;
    const uint64_t hs = dim / H, kvd = hs * c->n_kv_heads;
    /* Weights.init pointer carving, src/main.zig:85-112 */
    const float *p = data;
    m->token_embedding_table = p; p += V * dim;
    m->rms_att_weight = p;        p += L * dim;
    m->wq = p;                    p += L * dim * (H * hs);
    m->wk = p;                    p += L * dim * kvd;
    m->wv = p;                    p += L * dim * kvd;
    m->wo = p;                    p += L * (H * hs) * dim;
    m->rms_ffn_weight = p;        p += L * dim;
    m->w1 = p;                    p += L * dim * hid;
    m->w2 = p;                    p += L * hid * dim;
    m->w3 = p;                    p += L * dim * hid;
    m->rms_final_weight = p;      p += dim;
    m->freq_cis_real = p;         p += S * hs / 2;
    m->freq_cis_imag = p;         p += S * hs / 2;
    m->wcls = shared_weights ? m->token_embedding_table : p;
    /* RunState.init, src/main.zig:137-154 */
    m->x = orc_alloc(dim);   m->xb = orc_alloc(dim);  m->xb2 = orc_alloc(dim);
    m->hb = orc_alloc(hid);  m->hb2 = orc_alloc(hid);
    m->q = orc_alloc(dim);   m->k = orc_alloc(kvd);   m->v = orc_alloc(kvd);
    m->att = orc_alloc(H * S);
    m->logits = orc_alloc(V);
    m->key_cache = orc_alloc(L * S * kvd);
    m->value_cache = orc_alloc(L * S * kvd);
    if (!m->x || !m->xb || !m->xb2 || !m->hb || !m->hb2 || !m->q || !m->k || !m->v || !m->att ||
        !m->logits || !m->key_cache || !m->value_cache) {
        orc_model_destroy(m);
        return NULL;
    }
    return m;
}

void orc_model_destroy(orc_model *m) {
    if (!m) return;
    free(m->x); free(m->xb); free(m->xb2); free(m->hb); free(m->hb2); free(m->q); free(m->k);
    free(m->v); free(m->att); free(m->logits); free(m->key_cache); free(m->value_cache);
    free(m);
}

float *orc_logits(orc_model *m) { return m->logits; }

float *orc_state(orc_model *m, int which, uint64_t *len) {
    const orc_config *c = &m->cfg;
    const uint64_t dim = c->dim, hid = c->hidden_dim, L = c->n_layers, S = c->seq_len,
                   H = c->n_heads;
    const uint64_t kvd = dim / H * c->n_kv_heads;
    float *p = NULL;
    uint64_t n = 0;
    switch (which) {
    case 0: p = m->x; n = dim; break;
    case 1: p = m->xb; n = dim; break;
    case 2: p = m->xb2; n = dim; break;
    case 3: p = m->hb; n = hid; break;
    case 4: p = m->hb2; n = hid; break;
    case 5: p = m->q; n = dim; break;
    case 6: p = m->k; n = kvd; break;
    case 7: p = m->v; n = kvd; break;
    case 8: p = m->att; n = H * S; break;
    case 9: p = m->key_cache; n = L * S * kvd; break;
    case 10: p = m->value_cache; n = L * S * kvd; break;
    default: break;
    }
    if (len) *len = n;
    return p;
}

/* transformer(), src/main.zig:285-430. */
void orc_transformer(orc_model *m, int token, int pos) {
    const orc_config *c = &m->cfg;
    const int W = m->W;
    const int dim = c->dim, hidden_dim = c->hidden_dim;
    const int head_size = dim / c->n_heads;                       /* :289 */
    const int kv_dim = (dim * c->n_kv_heads) / c->n_heads;        /* :290 */
    const int kv_mul = c->n_heads / c->n_kv_heads;                /* :291 */
    float *x = m->x;

    memcpy(x, m->token_embedding_table + (size_t)token * dim, sizeof(float) * dim); /* :295-296 */

    for (int l = 0; l < c->n_layers; ++l) {                       /* :303 */
        orc_rmsnorm(m->xb, x, m->rms_att_weight + (size_t)l * dim, dim, W); /* :305 */

        const float *wq = m->wq + (size_t)l * dim * dim;
        const float *wk = m->wk + (size_t)l * dim * kv_dim;
        const float *wv = m->wv + (size_t)l * dim * kv_dim;
        if (kv_dim == dim) {                                      /* :308-313 */
            orc_matmul_fused3(m->q, m->k, m->v, m->xb, wq, wk, wv, dim, dim, W);
        } else {                                                  /* :314-320 */
            orc_matmul(m->q, m->xb, wq, dim, dim, W);
            orc_matmul_fused2(m->k, m->v, m->xb, wk, wv, kv_dim, dim, W);
        }

        for (int i = 0; i < dim; i += 2) {                        /* :336-351 */
            float fcr, fci;
            orc_rope_angle(i, head_size, pos, &fcr, &fci);
            const int rotn = (i < kv_dim) ? 2 : 1;                /* :343 */
            for (int v = 0; v < rotn; ++v) {
                float *vec = (v == 0) ? m->q : m->k;
                const float v0 = vec[i], v1 = vec[i + 1];
                vec[i] = v0 * fcr - v1 * fci;                     /* :348 */
                vec[i + 1] = v0 * fci + v1 * fcr;                 /* :349 */
            }
        }

        const size_t loff = (size_t)l * c->seq_len * kv_dim;      /* :354 */
        memcpy(m->key_cache + loff + (size_t)pos * kv_dim, m->k, sizeof(float) * kv_dim);
        memcpy(m->value_cache + loff + (size_t)pos * kv_dim, m->v, sizeof(float) * kv_dim);

        for (int h = 0; h < c->n_heads; ++h) {                    /* :361-389 */
            const float *q = m->q + (size_t)h * head_size;
            float *att = m->att + (size_t)h * c->seq_len;
            for (int t = 0; t <= pos; ++t) {
                const float *k = m->key_cache + loff + (size_t)t * kv_dim +
                                 (size_t)(h / kv_mul) * head_size;
                float score = orc_dot(q, k, head_size, W);
                score /= sqrtf((float)head_size);                 /* :372 */
                att[t] = score;
            }
            orc_softmax(att, pos + 1);                            /* :378 */
            orc_weighted_sum_rows(m->xb + (size_t)h * head_size, head_size,
                                  m->value_cache + loff + (size_t)(h / kv_mul) * head_size,
                                  kv_dim, att, pos + 1, W);       /* :381-388 */
        }

        orc_matmul(m->xb2, m->xb, m->wo + (size_t)l * dim * dim, dim, dim, W); /* :392 */
        orc_accum(x, m->xb2, dim);                                /* :395 */

        orc_rmsnorm(m->xb, x, m->rms_ffn_weight + (size_t)l * dim, dim, W);    /* :398 */

        orc_matmul_fused2(m->hb, m->hb2, m->xb, m->w1 + (size_t)l * dim * hidden_dim,
                          m->w3 + (size_t)l * dim * hidden_dim, hidden_dim, dim, W); /* :405-408 */
        for (int i = 0; i < hidden_dim; ++i)                      /* :411-413 */
            m->hb[i] = m->hb[i] * (1.0f / (1.0f + expf(-m->hb[i])));
        orc_vector_mul(m->hb, m->hb2, hidden_dim, W);             /* :416 */

        orc_matmul(m->xb, m->hb, m->w2 + (size_t)l * dim * hidden_dim, dim, hidden_dim, W); /* :419 */
        orc_accum(x, m->xb, dim);                                 /* :422 */
    }

    orc_rmsnorm(x, x, m->rms_final_weight, dim, W);               /* :426 */
    orc_matmul(m->logits, x, m->wcls, c->vocab_size, dim, W);     /* :429 */
}

static double orc_now(void) {
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

/* Generation loop at temperature 0, src/main.zig:995-1042 (printing omitted). */
int orc_generate(orc_model *m, int token0, int n_steps, const int32_t *forced, int stop_on_bos,
                 int32_t *out_next, double *secs_after_first) {
    int token = token0, pos = 0, calls = 0;
    double t0 = -1.0;
    if (n_steps > m->cfg.seq_len) n_steps = m->cfg.seq_len;       /* :993 */
    for (; pos < n_steps; ++pos) {
        orc_transformer(m, token, pos);                           /* :996 */
        ++calls;
        int next = forced ? forced[pos] : orc_argmax(m->logits, m->cfg.vocab_size);
        if (out_next) out_next[pos] = next;
        if (stop_on_bos && next == 1) break;                      /* :1017-1019 */
        token = next;
        if (t0 < 0.0) t0 = orc_now();                             /* :1038-1041 */
    }
    if (secs_after_first) *secs_after_first = (t0 < 0.0) ? 0.0 : orc_now() - t0;
    return calls;
}

/* ---- checkpoint file -------------------------------------------------------- */
int orc_read_header(const char *path, orc_config *cfg, int *shared_weights, uint64_t *file_floats) {
    FILE *f = fopen(path, "rb");
    if (!f) return -1;
    int32_t h[7];
    if (fread(h, sizeof(int32_t), 7, f) != 7) { fclose(f); return -2; }
    cfg->dim = h[0]; cfg->hidden_dim = h[1]; cfg->n_layers = h[2]; cfg->n_heads = h[3];
    cfg->n_kv_heads = h[4];
    if (shared_weights) *shared_weights = h[5] > 0;               /* :943 */
    cfg->vocab_size = h[5] < 0 ? -h[5] : h[5];                    /* :944 */
    cfg->seq_len = h[6];
    if (file_floats) {
        fseek(f, 0, SEEK_END);
        long sz = ftell(f);
        *file_floats = (uint64_t)(sz - 28) / 4;
    }
    fclose(f);
    return 0;
}

int orc_read_payload(const char *path, float *dst, uint64_t n) {
    FILE *f = fopen(path, "rb");
    if (!f) return -1;
    if (fseek(f, 28, SEEK_SET) != 0) { fclose(f); return -2; }
    size_t got = fread(dst, sizeof(float), n, f);
    fclose(f);
    return got == n ? 0 : -3;
}

/* ---- synthetic checkpoints --------------------------------------------------- */
static inline uint64_t orc_mix64(uint64_t z) {
    z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27; z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}

#define ORC_SYNTH_INV_STD 2.6428997921303014e-05 /* 1 / sqrt(4*(65536^2-1)/12) */

static void orc_synth_range(float *dst, uint64_t first, uint64_t count, uint64_t tensor_seed,
                            double mean, double scale, float lo, float hi) {
    for (uint64_t j = 0; j < count; ++j) {
        const uint64_t i = first + j;
        const uint64_t h = orc_mix64(tensor_seed + (i + 1) * 0x9E3779B97F4A7C15ull);
        const int32_t s = (int32_t)((h & 0xFFFF) + ((h >> 16) & 0xFFFF) + ((h >> 32) & 0xFFFF) +
                                    ((h >> 48) & 0xFFFF)) - 131070;
        volatile double prod = (double)s * scale; /* volatile: forbid a*b+c contraction */
        float v = (float)(prod + mean);
        if (v < lo) v = lo;
        if (v > hi) v = hi;
        dst[j] = v;
    }
}

typedef struct {
    float *dst; uint64_t first, count, seed; double mean, scale; float lo, hi;
} orc_synth_job;

static void *orc_synth_thread(void *arg) {
    orc_synth_job *j = (orc_synth_job *)arg;
    orc_synth_range(j->dst, j->first, j->count, j->seed, j->mean, j->scale, j->lo, j->hi);
    return NULL;
}

void orc_synth_fill(float *dst, uint64_t first, uint64_t count, uint64_t tensor_seed, double mean,
                    double sigma, float lo, float hi) {
    const double scale = sigma * ORC_SYNTH_INV_STD;
    enum { MAXT = 16 };
    long nproc = sysconf(_SC_NPROCESSORS_ONLN);
    int nt = (count < (1u << 20)) ? 1 : (int)(nproc < 1 ? 1 : (nproc > MAXT ? MAXT : nproc));
    if (nt == 1) {
        orc_synth_range(dst, first, count, tensor_seed, mean, scale, lo, hi);
        return;
    }
    pthread_t th[MAXT];
    orc_synth_job jobs[MAXT];
    const uint64_t chunk = (count + nt - 1) / nt;
    int started = 0;
    for (int t = 0; t < nt; ++t) {
        const uint64_t b = (uint64_t)t * chunk;
        if (b >= count) break;
        const uint64_t n = (b + chunk > count) ? count - b : chunk;
        jobs[t] = (orc_synth_job){dst + b, first + b, n, tensor_seed, mean, scale, lo, hi};
        if (pthread_create(&th[t], NULL, orc_synth_thread, &jobs[t]) != 0) {
            orc_synth_thread(&jobs[t]);
            th[t] = 0;
        }
        ++started;
    }
    for (int t = 0; t < started; ++t)
        if (th[t]) pthread_join(th[t], NULL);
}

void orc_synth_checkpoint(const orc_config *c, int shared_weights, uint64_t seed, float *data) {
    const uint64_t dim = c->dim, hid = c->hidden_dim, L = c->n_layers, V = c->vocab_size,
                   S = c->seq_len;
    const uint64_t hs = dim / c->n_heads, kvd = hs * c->n_kv_heads;
    const double sd = sqrt(288.0 / (double)dim), sh = sqrt(768.0 / (double)hid);
    const float BIG = 3.0e38f;
    float *p = data;
    int id = 0;
#define T(count, mean, sigma, lo, hi)                                                       \
    do {                                                                                    \
        orc_synth_fill(p, 0, (count), orc_mix64(seed * 1000003ull + (uint64_t)(++id)), (mean), \
                       (sigma), (lo), (hi));                                                \
        p += (count);                                                                       \
    } while (0)
    T(V * dim, 0.0, 0.04, -BIG, BIG);              /* 1 token_embedding_table */
    T(L * dim, 1.35, 0.35, 0.25f, 2.4f);           /* 2 rms_att_weight */
    T(L * dim * dim, 0.0, 0.04 * sd, -BIG, BIG);   /* 3 wq */
    T(L * dim * kvd, 0.0, 0.04 * sd, -BIG, BIG);   /* 4 wk */
    T(L * dim * kvd, 0.0, 0.02 * sd, -BIG, BIG);   /* 5 wv */
    T(L * dim * dim, 0.0, 0.02 * sd, -BIG, BIG);   /* 6 wo */
    T(L * dim, 1.35, 0.35, 0.25f, 2.4f);           /* 7 rms_ffn_weight */
    T(L * dim * hid, 0.0, 0.026 * sd, -BIG, BIG);  /* 8 w1 */
    T(L * hid * dim, 0.0, 0.026 * sh, -BIG, BIG);  /* 9 w2 */
    T(L * dim * hid, 0.0, 0.026 * sd, -BIG, BIG);  /* 10 w3 */
    T(dim, 7.1, 0.6, 3.0f, 10.0f);                 /* 11 rms_final_weight */
    memset(p, 0, sizeof(float) * (S * hs / 2) * 2); /* freq_cis_real/imag: unused (:67-69) */
    p += (S * hs / 2) * 2;
    id += 2;
    if (!shared_weights) T(V * dim, 0.0, 0.04, -BIG, BIG); /* 14 wcls */
#undef T
}
