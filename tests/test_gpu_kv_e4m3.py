"""GPU: the fp8 (e4m3) KV cache.  An e4m3-KV context returns exactly what an fp32-KV context of the same payload,
weight format, layout and scales returns when it stores every appended K/V value v as fl(e4m3(fl(v / s)) * s)
(kv_format "f32-round-e4m3", L2B_KV_ROUND_E4M3: its twin).

Each e4m3 kernel is the fp32 kernel the shape selects, with KV = e4m3: the QKV epilogue rounds each pair with
e4m3_round_bits under the layer's scale and stores it as one 16-bit word; the attention kernels load 4 bytes per
4 values, widen them exactly and multiply each by the scale in fp32.  The twin stores the same values widened
into its fp32 cache and reads them with the fp32 kernels.  Every comparison runs twice: with unit scales, and
with a stress scale set (stress_scales) under which at least 1% of layer 0's K codes saturate at +-448 and at
least 1% of its V codes are subnormal, which the tests assert.

  1  twin, bit for bit: every case of test_gpu_variants.CASES with fp32 weights, and bf16 and q8 weights on S
     and B: forward (logits, x, the widened caches), forward_argmax, forward_sample, generate_argmax, prefill,
     score; the batch, ragged and verify calls, generate_argmax_batch and fork on sessions;
     generate_speculative with the e4m3 cache on the target or on the draft; beam_search on paged models;
     the long-context shapes L7, L3 and F128 of test_gpu_long_context (L7 and L3 also under L2B_FUSE=0
     L2B_ATTN=3pass) on every path of its check_twin: forward at the checked positions, chunked prefill,
     score, the batch, ragged and verify calls at per-query T, forks.  The envelope shapes:
     test_gpu_envelope.test_envelope_kv.
  2  paged e4m3 against contiguous e4m3 (test_gpu_kv_paged's single-context check), and after forks,
     rewinds into shared pages (copies-on-write) and continuations.
  3  rounding: layer 0's K/V rows of an e4m3 context are round_e4m3_host of a plain fp32 context's layer-0
     rows under layer 0's scales, on the single step, the batched prefill, the batch and the ragged calls.
  4  stale rows: test_gpu_stale_rows' paths on e4m3 models (a NaN poison survives the rounding as 0x7F/0xFF).
  5  accounting and scales: kv_info, step_bytes, profile_step and page_bytes count 1 byte per element;
     sessions and forks take the format and the scales; l2b_kv_scales is refused after a session exists,
     after a step, on fp32 and bf16 KV models and with bad values, and a refused call changes no output.
  6  demo: with --kv-e4m3 the demo prints the text of Transformer(kv_format="e4m3")'s greedy tokens, and -v
     reports the model's and the draft's caches as e4m3.
"""
import os
import subprocess

import numpy as np
import pytest

import test_gpu_long_context as LC
from test_gpu_bf16 import _eq
from test_gpu_bf16_shapes import STALE_PATHS
from test_gpu_kv_bf16 import demo_text, layer0
from test_gpu_kv_paged import check_single as paged_check_single, rows, same_rows
from test_gpu_stale_rows import checkpoint, path_speculative, poison_token, stream_ends
from test_gpu_transformer import teacher_tokens
from test_gpu_variants import CASES, MODELS, l2b_env, payload
from test_gpu_verify_sample import host  # noqa: F401  (fixture)
from test_host_twin import tokenizer_path  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 64
SCALES = ["unit", "stress"]
F = np.float32


# ---- scales -------------------------------------------------------------------------------------------

_stress = {}
STRESS_ROWS = 258                              # stress_scales calibrates on the first min(seq_len, 258) rows


def stress_scales(l2b, ck, wf="f32", seed=None):
    """(n_layers, 2) scales from a plain fp32-KV context's caches after a prefill of the first positions:
    layer 0's s_k puts the top 3% of its |K| past 448 (saturated) and its s_v puts the bottom 3% of its
    nonzero |V| below 2^-6 (subnormal codes); the other layers are calibrated, amax / 448.  seed: the
    weights are device-synthesized."""
    key = (id(ck), wf, seed)
    if key not in _stress or _stress[key][0] is not ck:
        n = min(ck.seq_len, STRESS_ROWS)
        with l2b.Transformer(ck, seed, weight_format=wf) as f:
            f.prefill(teacher_tokens(n, ck.vocab_size), want_logits=False)
            K = np.abs(rows(f, "key_cache", n, ck))
            V = np.abs(rows(f, "value_cache", n, ck))
        s = np.empty((ck.n_layers, 2), F)
        for l in range(ck.n_layers):
            s[l] = K[l].max() / F(448), V[l].max() / F(448)
        s[0, 0] = np.quantile(K[0], 0.97) / F(448)
        s[0, 1] = np.quantile(V[0][V[0] > 0], 0.03) * F(64)
        assert np.all(np.isfinite(s)) and np.all(s > np.finfo(F).tiny), s
        _stress[key] = (ck, s)
    return _stress[key][1]


def scales_for(l2b, ck, which, wf="f32", seed=None):
    return np.ones((ck.n_layers, 2), F) if which == "unit" else stress_scales(l2b, ck, wf, seed)


def kv_pair(l2b, ck, scales, env=None, weight_format="f32", kv_layout="contiguous", seed=None):
    """(e4m3-KV context, its fp32-KV twin) of ck under env, both with `scales` (seed: device-synthesized
    weights)."""
    with l2b_env(env or {}):
        b = l2b.Transformer(ck, seed, weight_format=weight_format, kv_format="e4m3", kv_layout=kv_layout)
        f = l2b.Transformer(ck, seed, weight_format=weight_format, kv_format="f32-round-e4m3", kv_layout=kv_layout)
    b.set_kv_scales(scales)
    f.set_kv_scales(scales)
    return b, f


def check_edges(t, scales, n, what=""):
    """at least 1% of layer 0's first n K values saturated and of its V values subnormal (stress scales)"""
    k = rows(t, "key_cache", n, t.ck)[0]
    v = rows(t, "value_cache", n, t.ck)[0]
    sat = np.mean(np.abs(k) == F(448) * scales[0, 0])
    sub = np.mean((v != 0) & (np.abs(v) < F(2.0 ** -6) * scales[0, 1]))
    assert sat >= 0.01 and sub >= 0.01, (what, sat, sub)


def check_single(b, f, n, check, n_prompt, scales, stress):
    """The single-context entry points of b and its twin f over a teacher-forced run of n positions."""
    assert b.kv_info()[0] == "e4m3" and f.kv_info()[0] == "f32-round-e4m3"
    toks = teacher_tokens(n, b.ck.vocab_size)
    for pos, tok in enumerate(toks):
        lb, lf = b.forward(tok, pos), f.forward(tok, pos)
        if pos in check:
            _eq(lb, lf, f"logits at {pos}")
    for s in ("key_cache", "value_cache", "x", "logits"):
        _eq(b.state(s), f.state(s), s)
    if stress:
        check_edges(b, scales, n, "forward")
    for pos in check[:3]:
        assert b.forward_argmax(toks[pos], pos) == f.forward_argmax(toks[pos], pos)
    b.reset(); f.reset()
    forced = np.concatenate([np.array(toks[1:9], np.int32), np.full(8, -1, np.int32)])
    _eq(b.generate_argmax(toks[0], 0, 16, forced=forced, stop_on_bos=False),
        f.generate_argmax(toks[0], 0, 16, forced=forced, stop_on_bos=False), "generate_argmax")
    b.reset(); f.reset()
    _eq(b.prefill(toks[:n_prompt]), f.prefill(toks[:n_prompt]), "prefill logits")
    for s in ("key_cache", "value_cache"):
        _eq(b.state(s), f.state(s), f"prefill {s}")
    pb, cb = b.forward_sample(toks[n_prompt], n_prompt, 0.8, 0.9)
    pf, cf = f.forward_sample(toks[n_prompt], n_prompt, 0.8, 0.9)
    _eq(pb, pf, "forward_sample probs")
    assert (cb is None) == (cf is None) and (cb is None or np.array_equal(cb, cf))
    b.reset(); f.reset()
    lpb, gb = b.score(toks[:n_prompt])
    lpf, gf = f.score(toks[:n_prompt])
    _eq(lpb, lpf, "score log-probs")
    _eq(gb, gf, "score greedy")


# ---- 1: the twin --------------------------------------------------------------------------------------

@pytest.mark.parametrize("sc", SCALES)
@pytest.mark.parametrize("name,case,env", [(m, c, e) for m, c, e, _ in CASES],
                         ids=[f"{m}-{c}" for m, c, _, _ in CASES])
def test_twin(l2b, name, case, env, sc):
    _, _, n, check, n_prompt = MODELS[name]
    ck = payload(l2b, name)
    scales = scales_for(l2b, ck, sc)
    b, f = kv_pair(l2b, ck, scales, env)
    with b, f:
        check_single(b, f, n, check, n_prompt, scales, sc == "stress")


@pytest.mark.parametrize("sc", SCALES)
@pytest.mark.parametrize("wf", ["bf16", "q8"])
@pytest.mark.parametrize("name", ["S", "B"])
def test_twin_weight_formats(l2b, name, wf, sc):
    _, _, n, check, n_prompt = MODELS[name]
    ck = payload(l2b, name)
    scales = scales_for(l2b, ck, sc, wf)
    b, f = kv_pair(l2b, ck, scales, weight_format=wf)
    with b, f:
        assert b.weight_info()[0] == wf and f.weight_info()[0] == wf
        check_single(b, f, n, check, n_prompt, scales, sc == "stress")


@pytest.mark.parametrize("sc", SCALES)
@pytest.mark.parametrize("wf", ["f32", "bf16", "q8"])
@pytest.mark.parametrize("name", ["S", "B"])
def test_batched(l2b, name, wf, sc):
    ck = payload(l2b, name)
    b, f = kv_pair(l2b, ck, scales_for(l2b, ck, sc, wf), weight_format=wf)
    with b, f:
        toks = teacher_tokens(40, b.ck.vocab_size)
        sb = [b.session() for _ in range(4)]
        sf = [f.session() for _ in range(4)]
        try:
            assert all(s.kv_info()[0] == "e4m3" for s in sb) and all(s.kv_info()[0] == "f32-round-e4m3" for s in sf)
            for i in range(4):                           # sessions at different positions
                sb[i].prefill(toks[:3 + i], want_logits=False)
                sf[i].prefill(toks[:3 + i], want_logits=False)
            pos = [3, 4, 5, 6]
            t4 = toks[10:14]
            _eq(l2b.forward_batch(sb, t4, pos), l2b.forward_batch(sf, t4, pos), "forward_batch")
            pos = [p + 1 for p in pos]
            _eq(l2b.forward_argmax_batch(sb, t4, pos), l2b.forward_argmax_batch(sf, t4, pos), "argmax_batch")
            pos = [p + 1 for p in pos]
            rb = l2b.forward_sample_batch(sb, t4, pos, [1.0, 0.7, 1.0, 0.5], [0.9, 1.0, 0.95, 0.5])
            rf = l2b.forward_sample_batch(sf, t4, pos, [1.0, 0.7, 1.0, 0.5], [0.9, 1.0, 0.95, 0.5])
            _eq(rb[0], rf[0], "sample_batch probs")
            _eq(rb[2], rf[2], "sample_batch n_cand")
            pos = [p + 1 for p in pos]
            runs = [toks[0:1], toks[1:6], toks[6:9], toks[9:11]]     # NB 4 and NB 2 passes
            _eq(l2b.forward_ragged(sb, runs, pos), l2b.forward_ragged(sf, runs, pos), "forward_ragged")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            _eq(l2b.forward_argmax_ragged(sb, runs, pos), l2b.forward_argmax_ragged(sf, runs, pos), "argmax_ragged")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            rb = l2b.forward_sample_ragged(sb, runs, pos, [1.0] * 4, [0.9] * 4)
            rf = l2b.forward_sample_ragged(sf, runs, pos, [1.0] * 4, [0.9] * 4)
            _eq(rb[0], rf[0], "sample_ragged probs")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            gb = l2b.generate_argmax_batch(sb, t4, pos, 6, stop_on_bos=False)
            gf = l2b.generate_argmax_batch(sf, t4, pos, 6, stop_on_bos=False)
            for x, y in zip(gb, gf):
                _eq(x, y, "generate_argmax_batch")
            pos = [p + 6 for p in pos]
            vruns = [[int(g[-1])] + list(toks[20:23]) for g in gb]
            vb = l2b.verify_argmax_ragged(sb, vruns, pos)
            vf = l2b.verify_argmax_ragged(sf, vruns, pos)
            _eq(vb[1], vf[1], "n_accept")
            for x, y in zip(vb[0], vf[0]):
                _eq(x, y, "verify tokens")
            pos = [p + int(a) + 1 for p, a in zip(pos, vb[1])]
            wb = l2b.verify_sample_ragged(sb, vruns, pos, [1.0] * 4, [0.9] * 4)
            wf_ = l2b.verify_sample_ragged(sf, vruns, pos, [1.0] * 4, [0.9] * 4)
            _eq(wb[0], wf_[0], "verify_sample probs")
            _eq(wb[2], wf_[2], "verify_sample n_cand")
            for s in ("key_cache", "value_cache"):
                for x, y in zip(sb, sf):
                    _eq(x.state(s), y.state(s), f"session {s}")
            l2b.fork(sb[0], sb[1:], 5)
            l2b.fork(sf[0], sf[1:], 5)
            for s in ("key_cache", "value_cache"):
                for x, y in zip(sb[1:], sf[1:]):
                    _eq(x.state(s), y.state(s), f"forked {s}")
            assert all(s.kv_info()[0] == "e4m3" for s in sb)
            _eq(l2b.forward_batch(sb[1:], toks[30:33], [5, 5, 5]),
                l2b.forward_batch(sf[1:], toks[30:33], [5, 5, 5]), "after fork")
        finally:
            for s in sb + sf:
                s.close()


@pytest.mark.parametrize("sc", SCALES)
@pytest.mark.parametrize("name", ["S", "B"])
def test_speculative(l2b, name, sc):
    """generate_speculative with the e4m3 cache on the target (fp32-KV draft of another seed), and on the draft
    (fp32-KV target), against the same call with the reference cache in its place: the tokens, the rounds and
    the caches of target and draft, bit for bit."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = payload(l2b, name)
    dk = shape_checkpoint(MODELS[name][0])
    dk.data = l2b.synth_checkpoint_host(dk, MODELS[name][1] + 1000)
    for side in ("target", "draft"):
        kv = {"target": ("e4m3", "f32-round-e4m3"), "draft": ("f32", "f32")}
        dkv = {"target": ("f32", "f32"), "draft": ("e4m3", "f32-round-e4m3")}
        with l2b.Transformer(ck, kv_format=kv[side][0]) as tb, l2b.Transformer(ck, kv_format=kv[side][1]) as tf, \
                l2b.Transformer(dk, kv_format=dkv[side][0]) as db, l2b.Transformer(dk, kv_format=dkv[side][1]) as df:
            for t, c in ((tb, ck), (tf, ck), (db, dk), (df, dk)):
                if t.kv_info()[0] != "f32":
                    t.set_kv_scales(scales_for(l2b, c, sc))
            gb, rb = tb.generate_speculative(db, 1, 0, 24, 3, stop_on_bos=False)
            gf, rf = tf.generate_speculative(df, 1, 0, 24, 3, stop_on_bos=False)
            _eq(gb, gf, f"e4m3 cache on the {side}: tokens")
            assert rb == rf, (side, rb, rf)
            for s in ("key_cache", "value_cache"):
                _eq(tb.state(s), tf.state(s), f"e4m3 cache on the {side}: target {s}")
                _eq(db.state(s), df.state(s), f"e4m3 cache on the {side}: draft {s}")


@pytest.mark.parametrize("sc", SCALES)
@pytest.mark.parametrize("name", ["S", "B"])
def test_beam_search(l2b, name, sc):
    """beam_search on a paged e4m3 model and on its paged twin from the same prompt: tokens, log-probabilities,
    n_run and every beam's rows, bit for bit, at two prompt lengths with and without the BOS stop."""
    ck = payload(l2b, name)
    b, f = kv_pair(l2b, ck, scales_for(l2b, ck, sc), kv_layout="paged")
    toks = teacher_tokens(ck.seq_len, ck.vocab_size)
    with b, f:
        b.prefill(toks[:130], want_logits=False)
        f.prefill(toks[:130], want_logits=False)
        bb = [b.session() for _ in range(5)]
        bf = [f.session() for _ in range(5)]
        try:
            for pos, stop in ((127, True), (64, False)):
                rb = l2b.beam_search(b, toks[pos], pos, bb, 6, stop_on_bos=stop)
                rf = l2b.beam_search(f, toks[pos], pos, bf, 6, stop_on_bos=stop)
                assert rb[2] == rf[2]
                _eq(rb[1], rf[1], f"beam logprobs at {pos}")
                for i, (x, y) in enumerate(zip(rb[0], rf[0])):
                    _eq(x, y, f"beam {i} tokens at {pos}")
                    same_rows(bb[i], bf[i], pos + len(x), f"beam {i} at {pos}")
                for s in bb + bf:
                    s.reset()
        finally:
            for s in bb + bf:
                s.close()


@pytest.mark.parametrize("sc", SCALES)
@pytest.mark.parametrize("name,env_name", LC.TWIN_PARAMS)
def test_twin_long_context(l2b, name, env_name, sc):
    """The Llama head geometry at 4096 / 8192 positions on every path of test_gpu_long_context.check_twin:
    every split-count change, the switch to long chunks and the last positions (checked), teacher-forced,
    prefilled, scored, batched at per-query T and forked; attn_wo_kernel<4> (F128) and the 3-pass kernel."""
    ck = LC.payload(l2b, name)
    b, f = kv_pair(l2b, ck, scales_for(l2b, ck, sc), LC.ENVS[env_name])
    with b, f:
        LC.check_twin(l2b, b, f, name, env_name)


# ---- 2: paged against contiguous ----------------------------------------------------------------------

@pytest.mark.parametrize("sc", SCALES)
@pytest.mark.parametrize("wf", ["f32", "bf16"])
@pytest.mark.parametrize("name", ["S", "B"])
def test_paged(l2b, name, wf, sc):
    _, _, n, check, n_prompt = MODELS[name]
    ck = payload(l2b, name)
    scales = scales_for(l2b, ck, sc, wf)
    a = l2b.Transformer(ck, weight_format=wf, kv_format="e4m3", kv_layout="paged")
    b = l2b.Transformer(ck, weight_format=wf, kv_format="e4m3")
    with a, b:
        a.set_kv_scales(scales)
        b.set_kv_scales(scales)
        paged_check_single(a, b, n, check, n_prompt)


@pytest.mark.parametrize("sc", SCALES)
def test_paged_fork_and_copy_on_write(l2b, sc):
    """Forks share e4m3 pages; each destination continues with its own tokens, one rewinds into a shared page
    (copy-on-write); every session equals its contiguous e4m3 counterpart, src and siblings stay unchanged."""
    ck = payload(l2b, "S")
    scales = scales_for(l2b, ck, sc)
    a = l2b.Transformer(ck, kv_format="e4m3", kv_layout="paged")
    b = l2b.Transformer(ck, kv_format="e4m3")
    n_pos, rewind = 2 * P + 10, P + 20
    toks = teacher_tokens(n_pos + 8, ck.vocab_size)
    other = [int(t) for t in teacher_tokens(12, ck.vocab_size)[::-1]]
    with a, b:
        a.set_kv_scales(scales)
        b.set_kv_scales(scales)
        a.prefill(toks[:n_pos], want_logits=False)
        b.prefill(toks[:n_pos], want_logits=False)
        da = [a.session() for _ in range(3)]
        db = [b.session() for _ in range(3)]
        try:
            l2b.fork(a, da, n_pos)
            l2b.fork(b, db, n_pos)
            assert a.kv_pool_info()["pages_in_use"] == -(-n_pos // P) + 3 * (n_pos // P < -(-n_pos // P))
            for x, y in zip(da, db):
                same_rows(x, y, n_pos, "fork")
            _eq(da[0].prefill(other[:5], rewind), db[0].prefill(other[:5], rewind), "rewind into a shared page")
            same_rows(da[0], db[0], n_pos, "rewound destination")
            for i, (x, y) in enumerate(zip(da[1:], db[1:])):
                _eq(x.prefill(other[i:i + 3], n_pos), y.prefill(other[i:i + 3], n_pos), f"destination {i + 1}")
                same_rows(x, y, n_pos + 3, f"destination {i + 1}")
            same_rows(a, b, n_pos, "src")
            _eq(a.forward(toks[n_pos], n_pos), b.forward(toks[n_pos], n_pos), "src continues")
        finally:
            for s in da + db:
                s.close()


# ---- 3: rounding --------------------------------------------------------------------------------------

@pytest.mark.parametrize("sc", SCALES)
@pytest.mark.parametrize("name", ["S", "B"])
def test_rounding(l2b, name, sc):
    """Layer 0's K/V rows depend on the embedding and the weights alone, so they are round_e4m3_host of a plain
    fp32 context's rows, under layer 0's scales, on every path that appends them."""
    ck = payload(l2b, name)
    scales = scales_for(l2b, ck, sc)
    toks = teacher_tokens(40, ck.vocab_size)
    with l2b.Transformer(ck, kv_format="e4m3") as b, l2b.Transformer(ck) as f:
        b.set_kv_scales(scales)

        def same(x, y, what):
            for j, s in enumerate(("key_cache", "value_cache")):
                want = l2b.round_e4m3_host(np.ascontiguousarray(layer0(y, s)), scales[0, j])
                _eq(layer0(x, s), want, f"{what} {s}")
        for pos in range(5):                                  # the single step
            b.forward(toks[pos], pos); f.forward(toks[pos], pos)
        same(b, f, "forward")
        b.prefill(toks[5:21], 5, want_logits=False); f.prefill(toks[5:21], 5, want_logits=False)
        same(b, f, "prefill")
        sb, sf = [b.session() for _ in range(3)], [f.session() for _ in range(3)]
        try:
            l2b.forward_batch([b] + sb, toks[21:25], [21, 0, 0, 0])
            l2b.forward_batch([f] + sf, toks[21:25], [21, 0, 0, 0])
            same(b, f, "forward_batch")
            runs = [toks[22:30], toks[30:31], toks[31:33], toks[33:34]]
            l2b.forward_ragged([b] + sb, runs, [22, 1, 1, 1])
            l2b.forward_ragged([f] + sf, runs, [22, 1, 1, 1])
            same(b, f, "forward_ragged")
            for x, y in zip(sb, sf):
                same(x, y, "session")
        finally:
            for s in sb + sf:
                s.close()


# ---- 4: stale rows ------------------------------------------------------------------------------------

_poisoned = {}


@pytest.fixture(scope="module", autouse=True)
def _close_poisoned():
    yield
    for m, _, _ in _poisoned.values():
        m.close()
    _poisoned.clear()


def poisoned_kv_e4m3(l2b, oracle, name, wf, sc):
    key = (name, wf, sc)
    if key not in _poisoned:
        for m, _, _ in _poisoned.values():
            m.close()
        _poisoned.clear()
        ck = checkpoint(l2b, oracle, name)
        scales = scales_for(l2b, ck, sc, wf)
        P_ = poison_token(ck)
        data = ck.data.copy()
        data[P_ * ck.dim:(P_ + 1) * ck.dim] = np.nan
        pck = type(ck)(**{**ck.__dict__, "data": data})
        m = l2b.Transformer(pck, weight_format=wf, kv_format="e4m3")
        m.set_kv_scales(scales)
        s = m.session()
        try:                                   # the poison's rows are NaN codes, widened to NaN
            s.forward(P_, 0)
            assert np.isnan(rows(s, "key_cache", 1, ck)).all() and np.isnan(rows(s, "value_cache", 1, ck)).all()
        finally:
            s.close()
        _poisoned[key] = (m, ck, P_)
    return _poisoned[key]


@pytest.mark.parametrize("path", list(STALE_PATHS))
@pytest.mark.parametrize("wf,sc", [("f32", "unit"), ("bf16", "stress")])
@pytest.mark.parametrize("name", ["S", "B"])
def test_stale_rows(l2b, oracle, host, name, wf, sc, path):  # noqa: F811
    m, ck, P_ = poisoned_kv_e4m3(l2b, oracle, name, wf, sc)
    assert m.kv_info()[0] == "e4m3"
    ts = stream_ends(ck)
    if path == "speculative":
        path_speculative(l2b, host, m, P_, ts)
    else:
        STALE_PATHS[path](l2b, m, P_, ts)


# ---- 5: accounting and scales -------------------------------------------------------------------------

@pytest.mark.parametrize("wf", ["f32", "bf16", "q8"])
@pytest.mark.parametrize("name", ["S", "B"])
def test_accounting(l2b, name, wf):
    ck = payload(l2b, name)
    L, S = ck.n_layers, ck.seq_len
    kvd = ck.dim // ck.n_heads * ck.n_kv_heads
    with l2b.Transformer(ck, weight_format=wf, kv_format="e4m3") as b, l2b.Transformer(ck, weight_format=wf) as f, \
            l2b.Transformer(ck, weight_format=wf, kv_format="e4m3", kv_layout="paged") as p:
        assert b.kv_info() == ("e4m3", L * S * kvd * 2)
        assert f.kv_info() == ("f32", L * S * kvd * 2 * 4)
        assert b.weight_info() == f.weight_info()
        assert p.kv_pool_info()["page_bytes"] == 2 * L * P * kvd
        for pos in (0, 3, S - 1):
            wb, kb = b.step_bytes(pos)
            wf32, kf = f.step_bytes(pos)
            assert wb == wf32 and kb == L * 2 * kvd * (pos + 1) and kf == 4 * kb
        pb = {(n, l): by for n, l, _, by in b.profile_step(1, 0)}
        pf = {(n, l): by for n, l, _, by in f.profile_step(1, 0)}
        assert pb.keys() == pf.keys()
        for (n, l), by in pb.items():
            if n == "attention":
                assert by == 2 * kvd and pf[(n, l)] == 4 * by
            elif n == "attn_wo":
                assert pf[(n, l)] - by == 3 * 2 * kvd
            else:
                assert by == pf[(n, l)], (n, l)
        p.forward(1, 0)
        assert p.kv_info() == ("e4m3", 2 * L * P * kvd)
        s = b.session()
        try:
            assert s.kv_info() == b.kv_info() and s.weight_info() == b.weight_info()
        finally:
            s.close()


@pytest.mark.parametrize("name", ["S", "B"])
def test_sessions_and_forks_take_the_scales(l2b, name):
    ck = payload(l2b, name)
    scales = stress_scales(l2b, ck)
    toks = teacher_tokens(12, ck.vocab_size)
    with l2b.Transformer(ck, kv_format="e4m3") as b, l2b.Transformer(ck, kv_format="f32-round-e4m3") as f:
        b.set_kv_scales(scales)
        f.set_kv_scales(scales)
        s, d = b.session(), b.session()
        try:
            _eq(s.prefill(toks), f.prefill(toks), "a session of the scaled model")
            for x in (s, f):
                x.reset()
            s.prefill(toks, want_logits=False)
            l2b.fork(s, [d], 10)
            f.prefill(toks[:10], want_logits=False)
            same_rows(d, f, 10, "fork")
            _eq(d.forward(toks[10], 10), f.forward(toks[10], 10), "the fork continues")
            with l2b.Transformer(ck, kv_format="e4m3") as u:      # unit scales give other rows here
                u.prefill(toks[:10], want_logits=False)
                assert not np.array_equal(rows(u, "key_cache", 10, ck), rows(d, "key_cache", 10, ck))
        finally:
            s.close(); d.close()


def test_kv_scales_refusals(l2b):
    ck = payload(l2b, "S")
    L = ck.n_layers
    good = stress_scales(l2b, ck)
    toks = teacher_tokens(8, ck.vocab_size)

    def status(t, s):
        try:
            t.set_kv_scales(s)
            return 0
        except l2b.L2BError as e:
            return e.status
    with l2b.Transformer(ck, kv_format="e4m3") as ref:
        ref.set_kv_scales(good)
        want = ref.prefill(toks)
    with l2b.Transformer(ck, kv_format="e4m3") as b:
        assert status(b, good) == 0
        tiny = np.finfo(F).tiny
        for bad in (0.0, -1.0, np.inf, -np.inf, np.nan, tiny / 2):
            s = good.copy()
            s[L - 1, 1] = bad
            assert status(b, s) == -1, bad
        lib = b.lib
        from llama2_zig_b200.binding import FP
        flat = np.ascontiguousarray(good.ravel())
        for n in (0, 2 * L - 1, 2 * L + 1):
            assert lib.l2b_kv_scales(b.h, flat.ctypes.data_as(FP), n) == -1
        assert lib.l2b_kv_scales(b.h, None, 2 * L) == -1
        s = b.session()
        assert status(b, np.ones((L, 2), F)) == -7 and status(s, np.ones((L, 2), F)) == -7
        s.close()
        b.forward(toks[0], 0)
        assert status(b, np.ones((L, 2), F)) == -7
        b.reset()
        _eq(b.prefill(toks), want, "after the refused calls")
    for kv in ("f32", "bf16", "f32-round-bf16"):
        with l2b.Transformer(ck, kv_format=kv) as t:
            assert status(t, good) == -2, kv
    with l2b.Transformer(ck, kv_format="f32-round-e4m3") as t:
        assert status(t, good) == 0


# ---- 6: demo ------------------------------------------------------------------------------------------

def test_demo_kv_e4m3(l2b, stories15m, tokenizer_path):  # noqa: F811
    """--kv-e4m3 reaches the model and the draft (-v reports both caches as e4m3), and the demo prints the text
    of Transformer(kv_format="e4m3")'s greedy tokens on the same checkpoint: the host-argmax loop, the device
    loop and the drafted loop."""
    exe = os.path.join(ROOT, "llama2.zig_b200", "bin", "llama2_b200")
    base = [exe, stories15m, "-t", "0", "-n", "96", "-z", tokenizer_path, "--kv-e4m3", "-v"]
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    with l2b.Transformer(ck, kv_format="e4m3") as b:
        want = demo_text(tokenizer_path, b.generate_argmax(1, 0, 96, stop_on_bos=True))
        cache_bytes = b.kv_info()[1]
    assert len(want) > 0
    for extra in ([], ["--device-argmax"], ["--draft", stories15m]):
        r = subprocess.run(base + extra, capture_output=True, check=True, timeout=300)
        assert r.stdout.rstrip(b"\n") == want.rstrip(b"\n"), extra
        err = r.stderr.decode()
        assert f"kv cache: e4m3, {cache_bytes} bytes" in err.splitlines(), extra
        if extra[:1] == ["--draft"]:
            assert f"draft kv cache: e4m3, {cache_bytes} bytes" in err.splitlines()
