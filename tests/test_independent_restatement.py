"""CPU: a SECOND, independent restatement of transformer() (src/main.zig:285-430) in plain numpy
float64 — written from the reference text, sharing no code with oracle/ — reproduces the committed
golden token stream and agrees with the C oracle's logits.

Why: the reference has no test that pins transformer() and no Zig toolchain exists here (SURVEY 8c),
so the golden stream is derived.  Two restatements in different languages, arithmetic (fp64 vs the
reference's fp32 lane order) and authorship agreeing token for token — with a minimum top-2 margin
of 0.016 along the stream, ~10^4 x the reordering noise — is the strongest pin available offline
(ADVICE r1: "a shared misreading of main.zig would pass every test")."""
import hashlib
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rmsnorm(x, w):                                   # :432-468
    ss = np.mean(x * x) + 1e-5
    return x * (1.0 / np.sqrt(ss)) * w


class NumpyLlama:
    def __init__(self, ck):
        from llama2_zig_b200 import tp_plan
        self.ck = ck
        self.w = {k: np.asarray(v, dtype=np.float64) for k, v in tp_plan.payload_views(ck).items()}
        hs = ck.dim // ck.n_heads
        self.hs, self.kv_dim, self.kv_mul = hs, hs * ck.n_kv_heads, ck.n_heads // ck.n_kv_heads
        self.kc = np.zeros((ck.n_layers, ck.seq_len, self.kv_dim))
        self.vc = np.zeros_like(self.kc)

    def forward(self, token, pos):
        ck, w, hs = self.ck, self.w, self.hs
        x = w["token_embedding_table"][token].copy()                                  # :295-296
        i = np.arange(0, ck.dim, 2)
        freq = 1.0 / np.power(10000.0, (i % hs) / hs)                                 # :339
        c, s = np.cos(pos * freq), np.sin(pos * freq)                                 # :340-342
        for l in range(ck.n_layers):                                                  # :303
            xb = rmsnorm(x, w["rms_att_weight"][l])                                   # :305
            q, k, v = w["wq"][l] @ xb, w["wk"][l] @ xb, w["wv"][l] @ xb               # :308-320
            q0, q1 = q[0::2].copy(), q[1::2].copy()                                   # :346-349, adjacent pairs
            q[0::2], q[1::2] = q0 * c - q1 * s, q0 * s + q1 * c
            nk = self.kv_dim // 2                                                     # only i < kv_dim rotates k (:343)
            k0, k1 = k[0::2].copy(), k[1::2].copy()
            k[0::2], k[1::2] = k0 * c[:nk] - k1 * s[:nk], k0 * s[:nk] + k1 * c[:nk]
            self.kc[l, pos], self.vc[l, pos] = k, v                                   # :353-358
            out = np.zeros(ck.dim)
            for h in range(ck.n_heads):                                               # :361
                kvh = h // self.kv_mul
                keys = self.kc[l, :pos + 1, kvh * hs:(kvh + 1) * hs]
                att = keys @ q[h * hs:(h + 1) * hs] / np.sqrt(hs)                     # :367-375
                att = np.exp(att - att.max())
                att /= att.sum()                                                      # :378, :687-706
                out[h * hs:(h + 1) * hs] = att @ self.vc[l, :pos + 1, kvh * hs:(kvh + 1) * hs]   # :381-388
            x = x + w["wo"][l] @ out                                                  # :392-395
            xb = rmsnorm(x, w["rms_ffn_weight"][l])                                   # :398
            h1, h3 = w["w1"][l] @ xb, w["w3"][l] @ xb                                 # :405-408
            hb = h1 * (1.0 / (1.0 + np.exp(-h1))) * h3                                # :411-416
            x = x + w["w2"][l] @ hb                                                   # :419-422
        return w["wcls"] @ rmsnorm(x, w["rms_final_weight"])                          # :426-429


def test_numpy_restatement_reproduces_golden_stream_and_oracle_logits(l2b, oracle, stories15m):
    with open(os.path.join(GOLDEN, "stories15M_t0_tokens.json")) as f:
        gold = json.load(f)
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    m = NumpyLlama(ck)
    cfg, shared, data = oracle.read_checkpoint(stories15m)
    om = oracle.OracleModel(cfg, data, shared, W=8, kind="strict")
    token, toks, worst, min_margin = 1, [], 0.0, np.inf
    for pos in range(ck.seq_len):
        lg = m.forward(token, pos)
        if pos % 20 == 0 or pos > 215:
            want = om.forward(token, pos).astype(np.float64)
            worst = max(worst, float(np.max(np.abs(lg - want)) / np.max(np.abs(want))))
        else:
            om.forward(token, pos)
        top2 = np.partition(lg, -2)[-2:]
        min_margin = min(min_margin, float(top2[1] - top2[0]))
        nxt = int(np.argmax(lg))
        if nxt == 1:                                                                  # BOS ends the loop, :1017-1019
            break
        toks.append(nxt)
        token = nxt
    assert toks == gold["tokens"] and len(toks) == 256
    assert hashlib.sha256(np.array(toks, "<u4").tobytes()).hexdigest() == gold["sha256_le_u32"]
    assert worst <= 1e-5, worst                  # fp64 vs the fp32 lane-ordered oracle
    assert min_margin >= 0.015                   # 0.0166; see oracle_lib.STORIES15M_SEED
