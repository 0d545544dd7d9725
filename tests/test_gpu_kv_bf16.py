"""GPU: the bf16 KV cache.  A bf16-KV context returns exactly what an fp32-KV context of the same payload and
weight format returns when it rounds every appended K/V value to bf16 (kv_format "f32-round-bf16",
L2B_KV_ROUND_BF16: its twin).

Each bf16-KV kernel is the fp32 kernel the shape selects (the selection rules do not look at the cache
format), with KV = bf16: the QKV epilogue rounds each pair with bf16_round_bits and stores it as one 32-bit
word; the attention kernels load 8 bytes per 4 values and widen them exactly.  The twin stores the same
rounded values widened into its fp32 cache and reads them with the fp32 kernels.  So:

  1  twin, bit for bit: every case of test_gpu_variants.CASES with fp32 weights (flash NF family over head
     sizes 4..256, 3-pass, fused attn_wo_kernel, 32 splits, no graphs, batched GEMM against the position
     loop), and bf16 and q8 weights on S and B: forward (logits, x, the widened caches), forward_argmax,
     forward_sample, generate_argmax, prefill, score; the batch, ragged and verify calls,
     generate_argmax_batch and fork on sessions; generate_speculative with the bf16 cache on the target or
     on the draft (tokens, rounds and both caches); the long-context shapes L7, L3 and F128 of
     test_gpu_long_context (L7 and L3 also under L2B_FUSE=0 L2B_ATTN=3pass) on every path of its
     check_twin: forward at the checked positions, chunked prefill, score, the batch, ragged and verify
     calls at per-query T, forks.  The envelope shapes: test_gpu_envelope.test_envelope_kv.
  2  rounding: layer 0's K/V rows of a bf16-KV context are round_bf16_host of a plain fp32 context's layer-0
     rows, on the single step, the batched prefill, the batch and the ragged calls; every value read back
     has its low 16 bits zero.
  3  stale rows: test_gpu_stale_rows' paths on bf16-KV models with fp32 and bf16 weights (NaN survives the
     rounding); q8 with test_gpu_q8_shapes' other-stream fill.
  4  accounting: kv_info, step_bytes and profile_step count 2 bytes per cache element; weight_info does not
     see the flag; sessions and forks of a bf16-KV model are bf16-KV.
  5  demo: with --kv-bf16 the host loop, the device loop and the drafted loop print the text of
     Transformer(kv_format="bf16")'s greedy tokens on the same checkpoint, and -v reports the model's and
     the draft's caches as bf16.
"""
import os
import re
import struct
import subprocess

import numpy as np
import pytest

import test_gpu_long_context as LC
from test_gpu_bf16 import _eq
from test_gpu_bf16_shapes import STALE_PATHS
from test_gpu_q8_shapes import filled_session
from test_gpu_stale_rows import checkpoint, path_speculative, poison_token, stream_ends
from test_gpu_transformer import teacher_tokens
from test_gpu_variants import CASES, MODELS, l2b_env, payload
from test_gpu_verify_sample import host  # noqa: F401  (fixture)
from test_host_twin import tokenizer_path  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def kv_pair(l2b, ck, env=None, weight_format="f32", seed=None):
    """(bf16-KV context, its fp32-KV twin) of ck under env (seed: device-synthesized weights)."""
    with l2b_env(env or {}):
        b = l2b.Transformer(ck, seed, weight_format=weight_format, kv_format="bf16")
        f = l2b.Transformer(ck, seed, weight_format=weight_format, kv_format="f32-round-bf16")
    return b, f


def check_single(b, f, n, check, n_prompt):
    """The single-context entry points of b and its twin f over a teacher-forced run of n positions."""
    assert b.kv_info()[0] == "bf16" and f.kv_info()[0] == "f32-round-bf16"
    toks = teacher_tokens(n, b.ck.vocab_size)
    for pos, tok in enumerate(toks):
        lb, lf = b.forward(tok, pos), f.forward(tok, pos)
        if pos in check:
            _eq(lb, lf, f"logits at {pos}")
    for s in ("key_cache", "value_cache", "x", "logits"):
        _eq(b.state(s), f.state(s), s)
    assert not (b.state("key_cache").view(np.uint32) & 0xFFFF).any()
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


@pytest.mark.parametrize("name,case,env", [(m, c, e) for m, c, e, _ in CASES],
                         ids=[f"{m}-{c}" for m, c, _, _ in CASES])
def test_twin(l2b, name, case, env):
    _, _, n, check, n_prompt = MODELS[name]
    b, f = kv_pair(l2b, payload(l2b, name), env)
    with b, f:
        check_single(b, f, n, check, n_prompt)


@pytest.mark.parametrize("wf", ["bf16", "q8"])
@pytest.mark.parametrize("name", ["S", "B"])
def test_twin_weight_formats(l2b, name, wf):
    _, _, n, check, n_prompt = MODELS[name]
    b, f = kv_pair(l2b, payload(l2b, name), weight_format=wf)
    with b, f:
        assert b.weight_info()[0] == wf and f.weight_info()[0] == wf
        check_single(b, f, n, check, n_prompt)


@pytest.mark.parametrize("wf", ["f32", "bf16", "q8"])
@pytest.mark.parametrize("name", ["S", "B"])
def test_batched(l2b, name, wf):
    b, f = kv_pair(l2b, payload(l2b, name), weight_format=wf)
    with b, f:
        toks = teacher_tokens(40, b.ck.vocab_size)
        sb = [b.session() for _ in range(4)]
        sf = [f.session() for _ in range(4)]
        try:
            assert all(s.kv_info()[0] == "bf16" for s in sb) and all(s.kv_info()[0] == "f32-round-bf16" for s in sf)
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
            assert all(s.kv_info()[0] == "bf16" for s in sb)
            _eq(l2b.forward_batch(sb[1:], toks[30:33], [5, 5, 5]),
                l2b.forward_batch(sf[1:], toks[30:33], [5, 5, 5]), "after fork")
        finally:
            for s in sb + sf:
                s.close()


@pytest.mark.parametrize("wf", ["f32", "bf16"])
@pytest.mark.parametrize("name", ["S", "B"])
def test_speculative(l2b, name, wf):
    """generate_speculative with the bf16 cache on the target (fp32-KV draft of another seed), and on the draft
    (fp32-KV target), against the same call with the reference cache in its place: the tokens, the rounds
    (which depend on the draft's tokens) and the caches of target and draft, bit for bit."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = payload(l2b, name)
    dk = shape_checkpoint(MODELS[name][0])
    dk.data = l2b.synth_checkpoint_host(dk, MODELS[name][1] + 1000)
    for side in ("target", "draft"):
        kv = {"target": ("bf16", "f32-round-bf16"), "draft": ("f32", "f32")}
        dkv = {"target": ("f32", "f32"), "draft": ("bf16", "f32-round-bf16")}
        with l2b.Transformer(ck, weight_format=wf, kv_format=kv[side][0]) as tb, \
                l2b.Transformer(ck, weight_format=wf, kv_format=kv[side][1]) as tf, \
                l2b.Transformer(dk, weight_format=wf, kv_format=dkv[side][0]) as db, \
                l2b.Transformer(dk, weight_format=wf, kv_format=dkv[side][1]) as df:
            gb, rb = tb.generate_speculative(db, 1, 0, 24, 3, stop_on_bos=False)
            gf, rf = tf.generate_speculative(df, 1, 0, 24, 3, stop_on_bos=False)
            _eq(gb, gf, f"bf16 cache on the {side}: tokens")
            assert rb == rf, (side, rb, rf)
            for s in ("key_cache", "value_cache"):
                _eq(tb.state(s), tf.state(s), f"bf16 cache on the {side}: target {s}")
                _eq(db.state(s), df.state(s), f"bf16 cache on the {side}: draft {s}")


@pytest.mark.parametrize("name,env_name", LC.TWIN_PARAMS)
def test_twin_long_context(l2b, name, env_name):
    """The Llama head geometry at 4096 / 8192 positions on every path of test_gpu_long_context.check_twin:
    every split-count change, the switch to long chunks and the last positions (checked), teacher-forced,
    prefilled, scored, batched at per-query T and forked; attn_wo_kernel<4> (F128) and the 3-pass kernel."""
    ck = LC.payload(l2b, name)
    b, f = kv_pair(l2b, ck, LC.ENVS[env_name])
    with b, f:
        LC.check_twin(l2b, b, f, name, env_name)


def layer0(t, s):
    ck = t.ck
    kvd = ck.dim // ck.n_heads * ck.n_kv_heads
    return t.state(s).reshape(ck.n_layers, ck.seq_len, kvd)[0]


@pytest.mark.parametrize("name", ["S", "B"])
def test_rounding(l2b, name):
    """Layer 0's K/V rows depend on the embedding and the weights alone, so they are round_bf16_host of
    a plain fp32 context's rows on every path that appends them."""
    ck = payload(l2b, name)
    toks = teacher_tokens(40, ck.vocab_size)
    with l2b.Transformer(ck, kv_format="bf16") as b, l2b.Transformer(ck) as f:
        def same(what):
            for s in ("key_cache", "value_cache"):
                kb = layer0(b, s)
                assert not (kb.view(np.uint32) & 0xFFFF).any(), (what, s)
                _eq(kb, l2b.round_bf16_host(np.ascontiguousarray(layer0(f, s))), f"{what} {s}")
        for pos in range(5):                                  # the single step
            b.forward(toks[pos], pos); f.forward(toks[pos], pos)
        same("forward")
        b.prefill(toks[5:21], 5, want_logits=False); f.prefill(toks[5:21], 5, want_logits=False)
        same("prefill")
        sb, sf = [b.session() for _ in range(3)], [f.session() for _ in range(3)]
        try:
            l2b.forward_batch([b] + sb, toks[21:25], [21, 0, 0, 0])
            l2b.forward_batch([f] + sf, toks[21:25], [21, 0, 0, 0])
            same("forward_batch")
            runs = [toks[22:30], toks[30:31], toks[31:33], toks[33:34]]
            l2b.forward_ragged([b] + sb, runs, [22, 1, 1, 1])
            l2b.forward_ragged([f] + sf, runs, [22, 1, 1, 1])
            same("forward_ragged")
            for x, y in zip(sb, sf):
                for s in ("key_cache", "value_cache"):
                    _eq(layer0(x, s), l2b.round_bf16_host(np.ascontiguousarray(layer0(y, s))), f"session {s}")
        finally:
            for s in sb + sf:
                s.close()


# ---- stale rows ---------------------------------------------------------------------------------------

_poisoned = {}


@pytest.fixture(scope="module", autouse=True)
def _close_poisoned():
    yield
    for m, _, _ in _poisoned.values():
        m.close()
    _poisoned.clear()


def poisoned_kv_bf16(l2b, oracle, name, wf):
    key = (name, wf)
    if key not in _poisoned:
        for m, _, _ in _poisoned.values():
            m.close()
        _poisoned.clear()
        ck = checkpoint(l2b, oracle, name)
        P = poison_token(ck)
        data = ck.data.copy()
        data[P * ck.dim:(P + 1) * ck.dim] = np.nan
        pck = type(ck)(**{**ck.__dict__, "data": data})
        _poisoned[key] = (l2b.Transformer(pck, weight_format=wf, kv_format="bf16"), ck, P)
    return _poisoned[key]


@pytest.mark.parametrize("path", list(STALE_PATHS))
@pytest.mark.parametrize("wf", ["f32", "bf16"])
@pytest.mark.parametrize("name", ["S", "B"])
def test_stale_rows(l2b, oracle, host, name, wf, path):  # noqa: F811
    m, ck, P = poisoned_kv_bf16(l2b, oracle, name, wf)
    assert m.kv_info()[0] == "bf16"
    ts = stream_ends(ck)
    if path == "speculative":
        path_speculative(l2b, host, m, P, ts)
    else:
        STALE_PATHS[path](l2b, m, P, ts)


@pytest.mark.parametrize("name", ["S", "B"])
def test_stale_rows_q8(l2b, name):
    """A q8 model cannot hold a NaN embedding row: rows past each stream's end hold another stream's values."""
    ck = payload(l2b, name)
    V, T = ck.vocab_size, ck.seq_len
    toks = teacher_tokens(T + 1, V)
    ends = sorted({e for e in [1, 2, 3, 63, 64, 65, 127, 128, 129, 255, 256, 257, T - 1] if 0 < e < T})
    with l2b.Transformer(ck, weight_format="q8", kv_format="bf16") as m:
        for e in ends:
            a, b = filled_session(m, ck, toks), m.session()
            try:
                before = a.state("key_cache").copy()
                _eq(a.prefill(toks[:e]), b.prefill(toks[:e]), f"prefill to {e}")
                _eq(a.generate_argmax(toks[e], e, min(4, T - e), stop_on_bos=False),
                    b.generate_argmax(toks[e], e, min(4, T - e), stop_on_bos=False), f"generate from {e}")
                n = e + min(4, T - e)
                rows = a.state("key_cache").reshape(ck.n_layers, T, -1)
                _eq(rows[:, :n], b.state("key_cache").reshape(ck.n_layers, T, -1)[:, :n], f"appended rows to {n}")
                _eq(rows[:, n:], before.reshape(ck.n_layers, T, -1)[:, n:], f"rows past {n} kept")
            finally:
                a.close(); b.close()


# ---- accounting ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("wf", ["f32", "bf16", "q8"])
@pytest.mark.parametrize("name", ["S", "B"])
def test_accounting(l2b, name, wf):
    ck = payload(l2b, name)
    L, S = ck.n_layers, ck.seq_len
    kvd = ck.dim // ck.n_heads * ck.n_kv_heads
    with l2b.Transformer(ck, weight_format=wf, kv_format="bf16") as b, l2b.Transformer(ck, weight_format=wf) as f:
        assert b.kv_info() == ("bf16", L * S * kvd * 2 * 2)
        assert f.kv_info() == ("f32", L * S * kvd * 2 * 4)
        assert b.weight_info() == f.weight_info()
        for pos in (0, 3, S - 1):
            wb, kb = b.step_bytes(pos)
            wf32, kf = f.step_bytes(pos)
            assert wb == wf32 and kb == 2 * L * 2 * kvd * (pos + 1) and kf == 2 * kb
        pb = {(n, l): by for n, l, _, by in b.profile_step(1, 0)}
        pf = {(n, l): by for n, l, _, by in f.profile_step(1, 0)}
        assert pb.keys() == pf.keys()
        for (n, l), by in pb.items():
            if n == "attention":
                assert by == 2 * kvd * 2 and pf[(n, l)] == 2 * by
            elif n == "attn_wo":
                assert pf[(n, l)] - by == 2 * kvd * 2
            else:
                assert by == pf[(n, l)], (n, l)
        s = b.session()
        try:
            assert s.kv_info() == b.kv_info() and s.weight_info() == b.weight_info()
        finally:
            s.close()


# ---- demo ---------------------------------------------------------------------------------------------

def demo_text(tokenizer_path, tokens):
    """What the demo prints for a greedy stream from BOS (l2h_print_token, stopping at BOS): each token's bytes,
    a "<0xXX>" token as that byte, the leading space of the token after BOS dropped."""
    with open(tokenizer_path, "rb") as f:
        f.read(4)
        vocab = []
        while True:
            head = f.read(8)
            if len(head) < 8:
                break
            n = struct.unpack("<fi", head)[1]
            vocab.append(f.read(n))
    out, prev = b"", 1
    for t in tokens:
        if t == 1:
            break
        s = vocab[t]
        if prev == 1 and s[:1] == b" ":
            s = s[1:]
        m = re.fullmatch(rb"<0x([0-9A-Fa-f]{2})>", s)
        out += bytes([int(m.group(1), 16)]) if m else s
        prev = t
    return out


def test_demo_kv_bf16(l2b, stories15m, tokenizer_path):  # noqa: F811
    """--kv-bf16 reaches the model and the draft (-v reports both caches as bf16), and the demo prints the text
    of Transformer(kv_format="bf16")'s greedy tokens on the same checkpoint: the host-argmax loop, the device
    loop and the drafted loop."""
    exe = os.path.join(ROOT, "llama2.zig_b200", "bin", "llama2_b200")
    base = [exe, stories15m, "-t", "0", "-n", "96", "-z", tokenizer_path, "--kv-bf16", "-v"]
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    with l2b.Transformer(ck, kv_format="bf16") as b:
        want = demo_text(tokenizer_path, b.generate_argmax(1, 0, 96, stop_on_bos=True))
        cache_bytes = b.kv_info()[1]
    assert len(want) > 0
    for extra in ([], ["--device-argmax"], ["--draft", stories15m]):
        r = subprocess.run(base + extra, capture_output=True, check=True, timeout=300)
        assert r.stdout.rstrip(b"\n") == want.rstrip(b"\n"), extra
        err = r.stderr.decode()
        assert f"kv cache: bf16, {cache_bytes} bytes" in err.splitlines(), extra
        if extra[:1] == ["--draft"]:
            assert f"draft kv cache: bf16, {cache_bytes} bytes" in err.splitlines()
