"""GPU: long-context attention at the Llama head geometry (head size 128, 32 and 64 heads, 4096 and
8192 positions) on every decode, prefill and batched path, against the float64 forward pass of
tests/ref64.py.

Decode attention splits a query's timeline over `nsplit` CTAs per head.  create_run_state
(csrc/llama2_b200.cu) sets nsplit = min(ceil(2 SMs / heads), ceil(seq_len / 256), 32), and a query of
length T runs chunks of max(ceil(T / nsplit), 256) rows (`split_rows` restates both).  On a 132-SM
H100 with 32 heads that is 9 splits: up to T = 2304 the query runs ceil(T / 256) splits of 256 rows,
from T = 2305 on every split is longer than min_chunk and ends inside one of
attention_flash_kernel<4>'s 64-row passes (257 rows at T = 2305, 456 at 4096, 911 at 8192).  The
positions checked (`checked`) are derived from the device's own SM count: T = 1, 4, 256/257, 300, 512/513,
the last T with 256-row chunks and the one after it, the middle of the long-chunk regime and the
last 4 positions of the context.

Models (dim, hidden, layers, heads, kv_heads, vocab, seq_len); hidden and vocabulary are small, the
attention geometry is real.  The vocabularies are primes above seq_len, so the teacher tokens
(1 + 7919 p) % V never repeat:
  L7    (4096, 1376, 2, 32, 32, -4099, 4096)  llama2-7B attention, TMA ring, batched prefill.  Layer 1's
        KV rows depend on layer 0's attention at every position, so comparing them checks the
        batched prefill attention at all 4096 positions, not only at the checked ones.
  L3    (4096, 1376, 1, 32, 8, -8209, 8192)   Llama-3-8B: GQA 4, 911-row splits at T = 8192
  F128  (512, 1376, 2, 4, 2, -4099, 4096)     fused attn_wo_kernel<4> (default for dim <= 512), 8
        cluster splits of 512 rows at T = 4096; position-loop prefill
  L70   (8192, 1376, 1, 64, 8, -4099, 4096)   slow: 5 splits of 820 rows, gemv8_kernel, position-loop prefill
Weights: the synthetic payload; `sink` (test_ref64_cpu._key_spike on position 0 in every kv head: every
checked query of layer 0 puts > 0.99 of its weight on position 0, so every later split's max lies far
below the merged max); `peaked` (spikes 2 rows before the end of a checked T's query, one kv head per
spike: the spiked heads' max lies in the query's last split, more than PEAK_GAP above split 0's).
_key_spike's RoPE pair turns by up to 0.95 rad over 8192 positions at head size 128, so the sink spike
is raised to 80 (weight on position 0 at T = 8192: 1 - 1e-10), and both stresses are asserted on
the float64 run at the checked positions.
Environments: default everywhere; L2B_FUSE=0 L2B_ATTN=3pass (attention_kernel, score buffers of 456 /
911 rows, position-loop prefill) on L7 and L3.

Ledger: geometry / split regime / path / kernel -> test id (test_long_context[...])
  hs128 x 32 heads, 9 splits of 256 -> 911 rows, attention_flash_kernel<4>:
      teacher-forced forward, forward_argmax, forward_sample, generate_argmax     [L7-*-default], [L3-*-default]
      batched prefill (prefill_gemm_kernel + batched flash, per-query partials)  [L7-*-default], [L3-*-default]
      forward_batch / forward_ragged / verify_argmax_ragged (per-query T, pf_part_o / pf_part_ml / pf_counters)
                                                                                 [L7-*-default], [L3-*-default]
      score, fork                                                                every case
  GQA 4 at 8192 positions                                                        [L3-*]
  attention_kernel (3-pass), 456 / 911-row score buffers, position-loop prefill  [L7-*-3pass], [L3-*-3pass]
  attn_wo_kernel<4>, 8 cluster splits                                            [F128-*-default]
  64 heads, 5 splits of 820 rows, gemv8_kernel                                   [L70-*-default] (slow)

  KV caches (paged; bf16, e4m3 and their paged forms), bit for bit against their twins: check_twin, run
  by test_gpu_kv_paged, test_gpu_kv_bf16 and test_gpu_kv_e4m3 on L7, L3 and F128 (TWIN_PARAMS)

Bounds.  e(r) = max|r - ref64| / max|ref64| (log-probabilities: scaled by the position's max|logit|).
Every result is within REL_TOL = 1e-4, and within K[family, kernel class] * e_att.  The strict oracle
would take an hour per model at these sizes on a CPU host, so the yardstick is a float32 restatement
of attention at the checked rows only (`attention_yardstick`): float32 scores of the float64 run's
query and cache rows rounded to float32, the oracle's sequential `orc_softmax` and
`orc_weighted_sum_rows`, against ref64's attention output; e_att is its largest error over the
checked rows and layers of a checkpoint.  Measured e_dev / e_att on one H100 80GB HBM3 (max / median
over the cases; kernel classes: flash = attention_flash_kernel, fused = attn_wo_kernel, 3pass =
attention_kernel):
                      flash            fused            3pass
  logits              0.40 / 0.09      0.13 / 0.09      0.29 / 0.07
  KV rows             0.22 / 0.07      0.11 / 0.09      0.21 / 0.06
  score               0.16 / 0.03      0.07 / 0.02      0.14 / 0.02
  sample              6.29 / 0.07      0.20 / 0.06      6.29 / 0.04   (L3-sink: e = 6.3e-6)
e_att is floored at ATT_FLOOR = 1e-6 (sink's one-hot attention is exact to 3e-8 in float32).  The largest
error of any result is 6.3e-6.  K is 4x the worst ratio of its row, rounded up to an integer.  With every
attention score scaled by (1 + 2e-5) in attention_flash_kernel and attn_wo_kernel, the logits reach
2.8x (L7), 2.2x (L3) and 3.3x (F128) e_att and L7-peaked's KV rows 1.7x: L7-synthetic, L7-peaked,
L3-synthetic, F128-synthetic and F128-peaked fail the K bounds while every result stays within 1e-4.

Host cost: the file takes 328 s on one H100 80GB HBM3 (700 W), 277 s without the slow L70 cases.  The
host's share: payload synthesis, the float64 run and the yardstick take 24 s per L7 weight kind (layer
0's 4096-row attention as batched float64 matmuls), 4 s per L3 kind, 5 s per L70 kind and 2 s per
F128 kind on an 8-core CPU host, about 105 s for the whole file.
"""
import ctypes as C

import numpy as np
import pytest

import ref64
from test_gpu_ref64 import check_argmax, err, kv_rows
from test_gpu_transformer import REL_TOL, teacher_tokens
from test_gpu_variants import batched_prefill, l2b_env
from test_ref64_cpu import _key_spike, stress_check

pytestmark = pytest.mark.gpu

# name -> shape, synthetic seed, prefill path of the default environment (batched kernel or not)
MODELS = {"L7": ((4096, 1376, 2, 32, 32, -4099, 4096), 71, True),
          "L3": ((4096, 1376, 1, 32, 8, -8209, 8192), 73, True),
          "F128": ((512, 1376, 2, 4, 2, -4099, 4096), 75, False),
          "L70": ((8192, 1376, 1, 64, 8, -4099, 4096), 77, False)}
ENVS = {"default": {}, "3pass": {"L2B_FUSE": "0", "L2B_ATTN": "3pass"}}
KINDS = ("synthetic", "sink", "peaked")
CASES = [(m, k, e) for m in MODELS for k in KINDS for e in (("default", "3pass") if m in ("L7", "L3") else ("default",))]

MIN_CHUNK = 256                                    # AttnParams.min_chunk without L2B_ATTN_MIN_CHUNK
ATTN_CLUSTER = 8                                   # kAttnClusterCtas: attn_wo_kernel's splits per head
SINK_SPIKE = 80.0                                  # score raise of position 0's key
PEAK_SPIKE = 40.0                                  # score raise of a spiked key in the last split
PEAK_GAP = 20.0                                    # its split's max above split 0's

# (path family, kernel class) -> K, 4x the worst measured e_dev / e_att (module docstring)
K = {("logits", "flash"): 2, ("logits", "fused"): 1, ("logits", "3pass"): 2,
     ("kv", "flash"): 1, ("kv", "fused"): 1, ("kv", "3pass"): 1,
     ("score", "flash"): 1, ("score", "fused"): 1, ("score", "3pass"): 1,
     ("sample", "flash"): 26, ("sample", "fused"): 1, ("sample", "3pass"): 26}
FAMILY = {"forward": "logits", "prefill": "logits", "batch": "logits", "ragged": "logits",
          "kv": "kv", "prefill-kv": "kv", "ragged-kv": "kv", "score": "score", "sample": "sample"}

# floor of e_att: where a head's attention is one-hot (sink) the float32 attention is exact to 3e-8,
# while the GEMVs around it still round at ~1e-6
ATT_FLOOR = 1e-6

OBSERVED = []                                      # (path, case, kernel class, e_dev, e_att)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def split_rows(heads, seq_len, sms, T):
    """(nsplit, rows per split, active splits) of a query of length T: create_run_state's nsplit and
    attention_flash_kernel's chunk."""
    ns = min(-(-2 * sms // heads), -(-seq_len // MIN_CHUNK), 32)
    ns = max(ns, 1)
    chunk = max(-(-T // ns), MIN_CHUNK)
    return ns, chunk, -(-T // chunk)


def last_short(heads, seq_len, sms):
    """The last T whose splits are min_chunk rows long (T = 2304 at 9 splits).  Where the splits never
    grow past min_chunk before the context ends (F128's 16 splits of 4096), T = 2304: there
    attn_wo_kernel's 8 cluster splits are 288 rows long."""
    ns = split_rows(heads, seq_len, sms, 1)[0]
    return ns * MIN_CHUNK if ns * MIN_CHUNK + 8 < seq_len else 2304


def checked(shape, sms):
    """Positions p (T = p + 1) checked on a model: where the active split count changes, the switch to
    long chunks, the middle of the long-chunk regime, the last 4 positions."""
    heads, S = shape[3], shape[6]
    tl = last_short(heads, S, sms)
    ts = {1, 4, 256, 257, 300, 512, 513, tl, tl + 1, (tl + 1 + S) // 2, S - 3, S - 2, S - 1, S}
    return sorted(t - 1 for t in ts if 1 <= t <= S)


def peak_positions(shape, sms):
    """Spiked positions of `peaked`: 2 rows before each checked long-chunk query's end (the last 4
    positions share one), each in the last split of its query; at most one per kv head (F128 has 2)."""
    heads, S = shape[3], shape[6]
    tl = last_short(heads, S, sms)
    return [p for p in (S - 6, tl - 2, (tl + 1 + S) // 2 - 3) if p > 0][:shape[4]]   # one per kv head


_payloads, _refs = {}, {}


def payload(l2b, name):
    if name not in _payloads:
        from llama2_zig_b200.checkpoint import shape_checkpoint
        shape, seed, _ = MODELS[name]
        ck = shape_checkpoint(shape)
        ck.data = l2b.synth_checkpoint_host(ck, seed)
        _payloads.clear()
        _payloads[name] = ck
    return _payloads[name]


def weights(l2b, name, kind, sms):
    """(shape, float32 payload) of a model and weight kind."""
    shape = MODELS[name][0]
    data = payload(l2b, name).data
    if kind == "synthetic":
        return shape, data
    data = data.copy()
    w = ref64.tensors(shape, data)
    KV = shape[4]
    if kind == "sink":
        _key_spike(w, shape, 0, range(KV), SINK_SPIKE)
    else:
        for i, p in enumerate(peak_positions(shape, sms)):
            _key_spike(w, shape, p, [i % KV], PEAK_SPIKE)
    return shape, data


def query_split(shape, sms, T):
    """(rows per split, active splits) of a query of length T on the model's default attention
    kernel: attn_wo_kernel's ATTN_CLUSTER splits where it fuses (dim < 1024), else split_rows."""
    if shape[0] < 1024:
        chunk = -(-T // ATTN_CLUSTER)
        return chunk, -(-T // chunk)
    return split_rows(shape[3], shape[6], sms, T)[1:]


def peak_check(shape, run, sms):
    """In some head of layer 0 of every checked query with a spike in its last split (every
    long-chunk query, and on F128 all but the middle one), the max score lies in that split and
    exceeds split 0's max by more than PEAK_GAP."""
    heads, S = shape[3], shape[6]
    spikes = peak_positions(shape, sms)
    gaps = {}
    for p, sc in run.scores[0].items():
        chunk, active = query_split(shape, sms, p + 1)
        t0 = (active - 1) * chunk
        if active == 1 or not any(t0 <= q <= p for q in spikes):
            continue
        gaps[p] = max((float(sc[h, t0:].max() - sc[h, :chunk].max()) for h in range(heads)
                       if int(np.argmax(sc[h])) >= t0), default=-np.inf)
        assert gaps[p] > PEAK_GAP, (p, gaps[p])
    assert S - 1 in gaps and last_short(heads, S, sms) in gaps, sorted(gaps)
    return gaps


def attention_yardstick(oracle, shape, run):
    """Largest error, over the layers and checked rows of `run`, of a float32 attention against
    ref64's: float32 scores of the rounded query and cache rows, orc_softmax, orc_weighted_sum_rows."""
    lib = oracle.load("strict")
    dim, H, KV = shape[0], shape[3], shape[4]
    hs, kv_mul = dim // H, H // KV
    kv_dim = hs * KV
    root = np.float32(np.sqrt(np.float32(hs)))
    e = 0.0
    for l in run.att:
        for p, att in run.att[l].items():
            T = p + 1
            keys = run.key_cache[l, :T].astype(np.float32)
            vals = np.ascontiguousarray(run.value_cache[l, :T].astype(np.float32))
            q = run.q[l][p].astype(np.float32)
            out = np.zeros((H, hs), np.float32)
            for h in range(H):
                g = h // kv_mul
                sc = np.ascontiguousarray((keys[:, g * hs:(g + 1) * hs] @ q[h]) / root, dtype=np.float32)
                lib.orc_softmax(sc.ctypes.data_as(C.POINTER(C.c_float)), T)
                o = np.zeros(hs, np.float32)
                rows = C.cast(vals.ctypes.data + g * hs * 4, C.POINTER(C.c_float))
                lib.orc_weighted_sum_rows(o.ctypes.data_as(C.POINTER(C.c_float)), hs, rows, kv_dim,
                                          sc.ctypes.data_as(C.POINTER(C.c_float)), T, 8)
                out[h] = o
            e = max(e, err(out, att))
    return e


def reference(l2b, oracle, name, kind, sms):
    """(checkpoint, checked positions, ref64 run, e_att) of a model and weight kind, one at a time."""
    key = (name, kind)
    if key not in _refs:
        from llama2_zig_b200.checkpoint import shape_checkpoint
        _refs.clear()
        shape, data = weights(l2b, name, kind, sms)
        ck = shape_checkpoint(shape, data)
        check = checked(shape, sms)
        run = ref64.forward(shape, data, teacher_tokens(shape[6], ck.vocab_size), check)
        if kind == "sink":
            stress_check("sink", shape, run, shape[6])
        elif kind == "peaked":
            peak_check(shape, run, sms)
        _refs[key] = (ck, check, run, attention_yardstick(oracle, shape, run))
    return _refs[key]


def kernel_class(name, env_name):
    return "3pass" if env_name == "3pass" else "fused" if name == "F128" else "flash"


def bound(path, case, kclass, e_dev, e_att):
    OBSERVED.append((path, case, kclass, e_dev, e_att))
    assert e_dev <= REL_TOL, (path, e_dev)
    k = K[FAMILY[path], kclass]
    assert e_dev <= k * max(e_att, ATT_FLOOR), (path, e_dev, e_att, k)


# (model, environment) of the KV-cache twins (test_gpu_kv_paged, test_gpu_kv_bf16, test_gpu_kv_e4m3); the
# default environment's id is the model's name alone
TWIN_PARAMS = [pytest.param(m, e, id=m if e == "default" else f"{m}-{e}")
               for m in ("L7", "L3", "F128") for e in (("default", "3pass") if m != "F128" else ("default",))]


def check_twin(l2b, a, b, name, env_name):
    """a == b bit for bit, two contexts of model `name` created under ENVS[env_name] whose KV caches differ
    only in a way their contract says does not show (a paged context and its contiguous twin; a bf16 or
    e4m3 cache and the fp32 cache of its rounded values), on test_long_context's paths: teacher-forced
    forward at the checked positions, the caches below the appended count, the chunked prefill across
    last_short, score, forward_batch / forward_ragged / verify_argmax_ragged at per-query T, and forks at
    page-unaligned positions, the last one followed by decode steps."""
    from test_gpu_bf16 import _eq
    from test_gpu_kv_paged import same_rows
    sms = sm_count()
    ck = a.ck
    S = ck.seq_len
    check = checked(MODELS[name][0], sms)
    tl = last_short(ck.n_heads, S, sms)
    toks = teacher_tokens(S, ck.vocab_size)
    for pos, tok in enumerate(toks):
        la, lb = a.forward(tok, pos), b.forward(tok, pos)
        if pos in check:
            _eq(la, lb, f"logits at {pos}")
    same_rows(a, b, S, "forward")
    _eq(a.state("x"), b.state("x"), "x")
    for x in (a, b):
        x.reset()
    for lo, hi in zip([0, 37, tl - 1, tl + 2], [37, tl - 1, tl + 2, S]):
        _eq(a.prefill(toks[lo:hi], lo), b.prefill(toks[lo:hi], lo), f"prefill {lo}..{hi}")
    same_rows(a, b, S, "prefill")
    for x in (a, b):
        x.reset()
    for x, y, what in zip(a.score(toks), b.score(toks), ("log-probs", "greedy")):
        _eq(x, y, f"score {what}")                      # a and b now hold S - 1 positions

    with l2b_env(ENVS[env_name]):
        sa, sb = [a.session() for _ in range(3)], [b.session() for _ in range(3)]
    try:
        ta, tb = [a] + sa, [b] + sb
        ps = [S - 1, 3, 299, tl]                       # the sessions take 3, 299 and tl rows by fork
        for t in (ta, tb):
            for s, q in zip(t[1:], ps[1:]):
                l2b.fork(t[0], [s], q)
        _eq(l2b.forward_batch(ta, [toks[q] for q in ps], ps),
            l2b.forward_batch(tb, [toks[q] for q in ps], ps), "forward_batch")
        for x, y, q in zip(ta, tb, ps):
            same_rows(x, y, q + 1, "forward_batch")
        # session 1's prompt crosses tl / tl + 1 in chunks while the context decodes its last 3 positions
        cuts = [0, 37, tl - 1, tl + 1]
        for i in range(3):
            runs, pos = [toks[cuts[i]:cuts[i + 1]], [toks[S - 3 + i]]], [cuts[i], S - 3 + i]
            _eq(l2b.forward_ragged([ta[1], a], runs, pos), l2b.forward_ragged([tb[1], b], runs, pos),
                f"forward_ragged {i}")
        same_rows(ta[1], tb[1], tl + 1, "forward_ragged")
        same_rows(a, b, S, "forward_ragged")
        runs, pos = [toks[S - 4:S], toks[tl:tl + 1]], [S - 4, tl]
        va = l2b.verify_argmax_ragged([a, ta[3]], runs, pos)
        vb = l2b.verify_argmax_ragged([b, tb[3]], runs, pos)
        _eq(va[1], vb[1], "n_accept")
        for x, y in zip(va[0], vb[0]):
            _eq(x, y, "verify greedy")
        n_fork = 4000                                  # 62.5 pages of 64 rows
        for t in (ta, tb):
            l2b.fork(t[0], t[1:3], n_fork)
        for s, u in zip(ta[1:3], tb[1:3]):
            same_rows(s, u, n_fork, "fork")
            for q in range(n_fork, n_fork + 4):
                _eq(s.forward(toks[q], q), u.forward(toks[q], q), f"after the fork at {q}")
    finally:
        for s in sa + sb:
            s.close()


def test_split_rows_regimes():
    """split_rows at 132 SMs gives the regimes the module docstring names."""
    assert split_rows(32, 4096, 132, 2304) == (9, 256, 9)
    assert split_rows(32, 4096, 132, 2305) == (9, 257, 9)
    assert split_rows(32, 4096, 132, 4096) == (9, 456, 9)
    assert split_rows(32, 8192, 132, 8192) == (9, 911, 9)
    assert split_rows(64, 4096, 132, 4096) == (5, 820, 5)
    assert checked(MODELS["L7"][0], 132) == [0, 3, 255, 256, 299, 511, 512, 2303, 2304, 3199, 4092, 4093, 4094, 4095]


@pytest.mark.parametrize("name,kind,env_name",
                         [pytest.param(*c, marks=[pytest.mark.slow] if c[0] == "L70" else []) for c in CASES],
                         ids=[f"{m}-{k}-{e}" for m, k, e in CASES])
def test_long_context(l2b, oracle, name, kind, env_name):
    sms = sm_count()
    env = ENVS[env_name]
    shape = MODELS[name][0]
    assert batched_prefill(shape, env) == (MODELS[name][2] and env_name == "default")
    ck, check, run, e_att = reference(l2b, oracle, name, kind, sms)
    S = ck.seq_len
    case = f"{name}-{kind}-{env_name}"
    kclass = kernel_class(name, env_name)
    toks = teacher_tokens(S, ck.vocab_size)
    ref_k, ref_v = kv_rows(run.key_cache.reshape(-1), ck, S), kv_rows(run.value_cache.reshape(-1), ck, S)
    tl = last_short(ck.n_heads, S, sms)

    with l2b_env(env), l2b.Transformer(ck) as t:
        # teacher-forced forward over the whole context
        got = {}
        for pos, tok in enumerate(toks):
            lg = t.forward(tok, pos)
            if pos in check:
                got[pos] = lg
                bound("forward", case, kclass, err(lg, run.logits[pos]), e_att)
        dk, dv = kv_rows(t.state("key_cache"), ck, S), kv_rows(t.state("value_cache"), ck, S)
        bound("kv", case, kclass, err(dk, ref_k), e_att)
        bound("kv", case, kclass, err(dv, ref_v), e_att)

        for pos in check:
            check_argmax(t.forward_argmax(toks[pos], pos), got[pos], run.logits[pos])
        p = check[-1]
        for temp in (1.0, 0.6):
            probs, _ = t.forward_sample(toks[p], p, temp, 0.9)
            bound("sample", case, kclass, err(probs, ref64.softmax(run.logits[p] / temp)), e_att)

        t.reset()
        forced = np.array(toks[1:p + 1] + [-1], dtype=np.int32)
        out = t.generate_argmax(toks[0], 0, p + 1, forced=forced, stop_on_bos=False)
        assert out[:p].tolist() == toks[1:p + 1]
        check_argmax(int(out[p]), got[p], run.logits[p])

        # prefill in irregular chunks across the switch to long chunks: against float64 and against
        # the token-by-token run (bit for bit on the position loop, 1e-6 on the batched kernel)
        t.reset()
        cuts = [0, 37, tl - 1, tl + 2, S]
        for a, b in zip(cuts[:-1], cuts[1:]):
            lp = t.prefill(toks[a:b], a, want_logits=(b == S))
        bound("prefill", case, kclass, err(lp, run.logits[S - 1]), e_att)
        pk, pv = kv_rows(t.state("key_cache"), ck, S), kv_rows(t.state("value_cache"), ck, S)
        bound("prefill-kv", case, kclass, err(pk, ref_k), e_att)
        bound("prefill-kv", case, kclass, err(pv, ref_v), e_att)
        if batched_prefill(shape, env):
            assert err(lp, got[S - 1]) <= 1e-6
            for a, b in ((pk, dk), (pv, dv)):
                assert np.max(np.abs(a - b)) <= 1e-6 * np.max(np.abs(b))
        else:
            assert np.array_equal(lp, got[S - 1])
            assert np.array_equal(pk, dk) and np.array_equal(pv, dv)
        del pk, pv, dk, dv

        # score over the whole context
        t.reset()
        slp, greedy = t.score(toks)
        for pos in check:
            if pos + 1 >= S:
                continue
            z = run.logits[pos]
            scale = float(np.max(np.abs(z)))
            bound("score", case, kclass, abs(float(slp[pos]) - ref64.log_softmax(z)[toks[pos + 1]]) / scale, e_att)
            check_argmax(int(greedy[pos]), got[pos], z)

        sess = [t] + [t.session() for _ in range(3)]
        try:
            # forward_batch: queries at T = 4, 300, the first long-chunk T and seq_len
            ps = [3, 299, tl, S - 1]
            assert all(q in check for q in ps)
            for s, q in zip(sess, ps):
                s.reset()
                s.prefill(toks[:q], 0, want_logits=False)
            out = l2b.forward_batch(sess, [toks[q] for q in ps], ps)
            for row, q in zip(out, ps):
                bound("batch", case, kclass, err(row, run.logits[q]), e_att)

            # forward_ragged: session 0's prompt crosses tl / tl + 1 in chunks while session 1 decodes
            # the last 3 positions of the context
            cuts = [0, 37, tl - 1, tl + 1]
            for s in sess[:2]:
                s.reset()
            b0 = S - 3
            sess[1].prefill(toks[:b0], 0, want_logits=False)
            for i in range(3):
                out = l2b.forward_ragged(sess[:2], [toks[cuts[i]:cuts[i + 1]], [toks[b0 + i]]], [cuts[i], b0 + i])
            bound("ragged", case, kclass, err(out[0], run.logits[tl]), e_att)
            bound("ragged", case, kclass, err(out[1], run.logits[S - 1]), e_att)
            for c, r in ((t.state("key_cache"), ref_k), (t.state("value_cache"), ref_v)):
                bound("ragged-kv", case, kclass, err(kv_rows(c, ck, tl + 1), r[:, :tl + 1]), e_att)

            # verify_argmax_ragged: teacher drafts whose last one sits at seq_len - 1
            v0 = S - 4
            for s in sess[:2]:
                s.reset()
            sess[0].prefill(toks[:v0], 0, want_logits=False)
            sess[1].prefill(toks[:tl], 0, want_logits=False)
            greedy, n_acc = l2b.verify_argmax_ragged(sess[:2], [toks[v0:S], toks[tl:tl + 1]], [v0, tl])
            for g, start in ((greedy[0], v0), (greedy[1], tl)):
                for i, tok in enumerate(g):
                    check_argmax(int(tok), got[start + i], run.logits[start + i])
            dev_next = [int(np.argmax(got[v0 + i])) for i in range(3)]
            want_acc = next((i for i in range(3) if dev_next[i] != toks[v0 + 1 + i]), 3)
            assert int(n_acc[0]) == want_acc and int(n_acc[1]) == 0

            # fork of a 4000-row prefix to 3 sessions, then decode: bitwise a session that prefilled it
            n_fork = 4000
            t.reset()
            t.prefill(toks[:n_fork], 0, want_logits=False)
            l2b.fork(t, sess[1:], n_fork)
            base = [t.forward(toks[q], q) for q in range(n_fork, n_fork + 4)]
            for s in sess[1:]:
                for i, q in enumerate(range(n_fork, n_fork + 4)):
                    assert np.array_equal(s.forward(toks[q], q), base[i]), q
        finally:
            for s in sess[1:]:
                s.close()
