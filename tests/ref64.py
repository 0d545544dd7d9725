"""A float64 forward pass of transformer() (src/main.zig:285-430) over a teacher-forced run.

Written from the reference text alone, as a yardstick that shares no code and no reading with the C
oracle (oracle/llama2_oracle.c) or the library: it imports neither of them, nor the package's
payload views (tp_plan), and it finds every tensor in the checkpoint payload itself (the layout of
Weights.init, src/main.zig:73-115).  Every product, sum, norm and exponential is float64.  The
RoPE angle is the one exception: the reference computes it in f32 (:338-340: head_dim, freq and
pos * freq are f32 values), so that angle is part of what transformer() means; it is formed here
with the same f32 operations, and only its cos / sin are taken in float64.

A run is evaluated position-parallel (all positions of a layer at once, causal attention), which is
the same arithmetic as one position after another: position p reads only the cache rows 0..p.
"""
import numpy as np

NORM_EPS = 1e-5                                   # :432-468


def payload_layout(shape):
    """{tensor name: (offset in floats, shape)} of a payload after the 28-byte header, for the header
    tuple `shape` = (dim, hidden, layers, heads, kv_heads, vocab, seq_len): a negative vocab means an
    unshared classifier, stored after the two unused freq_cis blocks (:85-112, :943-944)."""
    dim, hid, L, H, KV, V, S = shape
    shared, V = V > 0, abs(V)
    hs = dim // H
    kv_dim = hs * KV
    parts = [("token_embedding_table", (V, dim)),
             ("rms_att_weight", (L, dim)),
             ("wq", (L, H * hs, dim)),
             ("wk", (L, kv_dim, dim)),
             ("wv", (L, kv_dim, dim)),
             ("wo", (L, dim, H * hs)),
             ("rms_ffn_weight", (L, dim)),
             ("w1", (L, hid, dim)),
             ("w2", (L, dim, hid)),
             ("w3", (L, hid, dim)),
             ("rms_final_weight", (dim,)),
             ("freq_cis_real", (S, hs // 2)),
             ("freq_cis_imag", (S, hs // 2))]
    if not shared:
        parts.append(("wcls", (V, dim)))
    out, off = {}, 0
    for name, shp in parts:
        out[name] = (off, shp)
        off += int(np.prod(shp))
    if shared:
        out["wcls"] = out["token_embedding_table"]                                    # :112
    out["_total"] = (off, ())
    return out


def payload_floats(shape):
    return payload_layout(shape)["_total"][0]


def tensors(shape, data):
    """Views of the float32 payload `data` by tensor name (no copies)."""
    lay = payload_layout(shape)
    assert data.size >= lay["_total"][0], (data.size, lay["_total"][0])
    return {k: data[o:o + int(np.prod(s))].reshape(s) for k, (o, s) in lay.items() if k != "_total"}


def rope_angles(positions, head_size):
    """(n, head_size/2) float64 cos and sin of the reference's f32 angle pos * freq (:336-342); pair j
    of a head is dims (2j, 2j+1) of that head, its head_dim is 2j."""
    hd = np.arange(0, head_size, 2, dtype=np.float32)
    freq = np.float32(1.0) / np.power(np.float32(10000.0), hd / np.float32(head_size))
    val = np.asarray(positions, dtype=np.float32)[:, None] * freq[None, :]
    val = val.astype(np.float64)
    return np.cos(val), np.sin(val)


def rmsnorm(x, w):                                 # :432-468, rows of x
    ss = np.mean(x * x, axis=-1, keepdims=True) + NORM_EPS
    return x / np.sqrt(ss) * w


def matmul(x, w, rows=8192):
    """x (n, k) float64 times w (d, k) float32, transposed: (n, d).  W is converted to float64 in
    slices of `rows` rows so a large classifier never exists twice in memory."""
    out = np.empty((x.shape[0], w.shape[0]))
    for r in range(0, w.shape[0], rows):
        out[:, r:r + rows] = x @ w[r:r + rows].astype(np.float64).T
    return out


def rotate(v, cos, sin):
    """Rotate adjacent pairs of every head of v (n, heads, hs) by the per-position angles (:344-350)."""
    v0, v1 = v[..., 0::2].copy(), v[..., 1::2].copy()
    c, s = cos[:, None, :], sin[:, None, :]
    v[..., 0::2] = v0 * c - v1 * s
    v[..., 1::2] = v0 * s + v1 * c
    return v


class Run:
    """What one teacher-forced run of tokens[0..n) at positions 0..n-1 leaves.

      logits[p], x[p] (after the final rmsnorm, :426), resid[p] (the residual stream before it) for
      every requested position p; key_cache, value_cache: (layers, seq_len, kv_dim) float64 with
      rows 0..n-1 filled, as state.key_cache / value_cache (:151-152, :353-358); probs[l][p]:
      (heads, p+1) attention weights of layer l at the requested positions, and scores[l][p] the
      scaled scores they come from (:367-378)."""

    def __init__(self):
        self.logits, self.x, self.resid, self.probs, self.scores = {}, {}, {}, {}, {}
        self.key_cache = self.value_cache = None


def forward(shape, data, tokens, want, block=1 << 22):
    """transformer(tokens[p], p) for p = 0 .. len(tokens)-1 (src/main.zig:285-430) in float64.

    `shape` is the header tuple (negative vocab: unshared classifier), `data` the float32 payload.
    Outputs are kept for the positions in `want`.  `block` bounds the attention score tile (heads x
    query rows x keys) in elements."""
    dim, hid, L, H, KV, V, S = shape
    V = abs(V)
    hs, kv_mul = dim // H, H // KV
    kv_dim = hs * KV
    w = tensors(shape, data)
    n = len(tokens)
    assert 0 < n <= S
    want = sorted(set(int(p) for p in want))
    assert all(0 <= p < n for p in want)
    cos, sin = rope_angles(np.arange(n), hs)
    r = Run()
    r.key_cache, r.value_cache = np.zeros((L, S, kv_dim)), np.zeros((L, S, kv_dim))
    x = w["token_embedding_table"][np.asarray(tokens)].astype(np.float64)          # :295-296
    rows = np.arange(n)
    for l in range(L):                                                             # :303
        xb = rmsnorm(x, w["rms_att_weight"][l].astype(np.float64))                 # :305
        k = matmul(xb, w["wk"][l]).reshape(n, KV, hs)                              # :308-320
        v = matmul(xb, w["wv"][l])
        rotate(k, cos, sin)                        # k's dims are all < kv_dim: every pair rotates (:343)
        r.key_cache[l, :n] = k.reshape(n, kv_dim)                                  # :353-358
        r.value_cache[l, :n] = v
        if l == L - 1:                             # past the last cache write only `want` rows matter
            rows = np.asarray(want)
            x, xb = x[rows], xb[rows]
        q = matmul(xb, w["wq"][l]).reshape(len(rows), H, hs)
        rotate(q, cos[rows], sin[rows])
        keys = r.key_cache[l, :n].reshape(n, KV, hs)
        vals = r.value_cache[l, :n].reshape(n, KV, hs)
        att_out = np.empty((len(rows), H, hs))
        step = max(1, block // (H * n))
        for b in range(0, len(rows), step):                                        # :361-389
            qb = q[b:b + step].reshape(-1, KV, kv_mul, hs)                         # head h reads kv head h / kv_mul
            sc = np.einsum("qgmd,tgd->qgmt", qb, keys) / np.sqrt(hs)                # :367-375
            pos = rows[b:b + step]
            sc = np.where(np.arange(n)[None, None, None, :] <= pos[:, None, None, None], sc, -np.inf)
            p = np.exp(sc - sc.max(axis=-1, keepdims=True))                        # :378, :687-706
            p /= p.sum(axis=-1, keepdims=True)
            att_out[b:b + step] = np.einsum("qgmt,tgd->qgmd", p, vals).reshape(-1, H, hs)   # :381-388
            for i, ps in enumerate(pos):
                if ps in want:
                    r.scores.setdefault(l, {})[int(ps)] = sc[i].reshape(H, n)[:, :ps + 1].copy()
                    r.probs.setdefault(l, {})[int(ps)] = p[i].reshape(H, n)[:, :ps + 1].copy()
        x = x + matmul(att_out.reshape(len(rows), dim), w["wo"][l])               # :392-395
        xb = rmsnorm(x, w["rms_ffn_weight"][l].astype(np.float64))                # :398
        h1, h3 = matmul(xb, w["w1"][l]), matmul(xb, w["w3"][l])                    # :405-408
        hb = h1 * (1.0 / (1.0 + np.exp(-h1))) * h3                                 # :411-416
        x = x + matmul(hb, w["w2"][l])                                             # :419-422
    xf = rmsnorm(x, w["rms_final_weight"].astype(np.float64))                     # :426
    logits = matmul(xf, w["wcls"])                                                 # :429
    for i, p in enumerate(want):
        r.logits[p], r.x[p], r.resid[p] = logits[i], xf[i], x[i]
    return r


def log_softmax(z):
    z = np.asarray(z, dtype=np.float64)
    m = np.max(z)
    return z - m - np.log(np.sum(np.exp(z - m)))


def softmax(z):
    return np.exp(log_softmax(z))
