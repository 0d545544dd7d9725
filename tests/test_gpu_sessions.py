"""GPU: sessions on one loaded model (l2b_create_session) and one step of several sessions per call
(l2b_forward_batch / l2b_forward_argmax_batch).

A session is a decode stream on the weights of a model, with its own KV cache and run state.  On the
shapes where l2b_prefill batches (pf_prepare in csrc/llama2_b200.cu), l2b_forward_batch runs up to 4
sessions per pass over the weights with the batched prefill's kernels, each vector at its own position
on its own cache, and a batched classifier.  Elsewhere it steps the sessions one after another.  The
checks here:

  * a session equals, bit for bit, an independent context of the same weights fed the same tokens, and
    leaves the model's own cache alone; its load_stats report 0 bytes;
  * the batched step equals the same sessions stepped one by one with l2b_forward: within 1e-6 on the
    batched kernels, bit for bit on the fallback; the launch count shows which path ran; the sessions
    start at staggered positions (prefilled), so one group mixes queries with 1 and 2 attention splits;
  * forward_argmax_batch == the first-index np.argmax of forward_batch's logits, also on the crafted
    classifiers of test_gpu_variants.test_device_argmax_edges;
  * refused calls (duplicate session, two models, position past the cache, token out of range) return
    their code and leave every cache unchanged;
  * destroying the model before its sessions: they keep stepping, and the device memory comes back
    after the last one;
  * both sides of the batched budget (test_gpu_envelope's pf-hid19840 / pf-hid19844), and llama2-7B at
    full depth with 4 sessions where 4 contexts would not fit (slow).

Ledger: kernel instantiation -> a test that runs it
  prefill_gemm_kernel<QKV, 4> with per-vector positions and caches, <SILU, 4>, <RESID, 4>, <RESID, 2>
                                             test_batch_equals_single_steps[B-*], test_batch_envelope[pf-hid19840]
  prefill_gemm_kernel<STORE, 4>              test_batch_equals_single_steps[B-*] (odd 32003-row vocabulary)
  prefill_gemm_kernel<ARGMAX, 4>             test_batch_equals_single_steps[B-*], test_batch_argmax_edges[*]
  prefill_gemm_kernel<STORE | ARGMAX, 2>     instantiated by pf_pick<2>, never launched (the classifier's
                                             input is dim-wide: 4 per pass)
  attention_flash_kernel<2>, batched, per-query position / cache / split count
                                             test_batch_equals_single_steps[B-*]
  fallback (each session's own step graph)   test_batch_equals_single_steps[S-*], [B-prefill-batch0-*],
                                             test_batch_envelope[pf-hid19844]
"""
import numpy as np
import pytest

from test_gpu_envelope import ENVELOPE
from test_gpu_transformer import REL_TOL, rel_err, teacher_tokens
from test_gpu_variants import MODELS, batched_prefill, crafted, l2b_env, oracle_ref, payload

pytestmark = pytest.mark.gpu


def stream(b, n, vocab):
    """Teacher-forced tokens of session b (session 0: teacher_tokens, which the oracle runs)."""
    return [(1 + 7919 * p + 104729 * b) % vocab for p in range(n)]


def batch_launches(n_layers, n):
    """Kernels of one batched step of n sessions: per group of up to 4, per layer qkv, attention, wo,
    w13 and one w2 per pair, then the classifier."""
    groups = [min(4, n - g) for g in range(0, n, 4)]
    return sum(n_layers * (4 + (nb + 1) // 2) + 1 for nb in groups)


def caches(t):
    return t.state("key_cache"), t.state("value_cache")


def close_all(ts):
    for t in ts:
        t.close()


@pytest.mark.parametrize("name", ["B", "S"])
def test_sessions_match_independent_contexts(l2b, name):
    ck = payload(l2b, name)
    V, n = ck.vocab_size, 40
    with l2b_env({}), l2b.Transformer(ck) as m:
        for pos, tok in enumerate(teacher_tokens(5, V)):
            m.forward(tok, pos)
        km, vm = caches(m)
        a, b = m.session(), m.session()
        ta, tb = l2b.Transformer(ck), l2b.Transformer(ck)
        try:
            assert a.load_stats()[1] == 0 and b.load_stats()[1] == 0 and m.load_stats()[1] > 0
            sa, sb = stream(1, n, V), stream(2, n, V)
            for pos in range(n):
                la, lb = a.forward(sa[pos], pos), b.forward(sb[pos], pos)
                assert np.array_equal(la, ta.forward(sa[pos], pos)), pos
                assert np.array_equal(lb, tb.forward(sb[pos], pos)), pos
            for s, t in ((a, ta), (b, tb)):
                for x, y in zip(caches(s), caches(t)):
                    assert np.array_equal(x, y)
            for x, y in zip(caches(m), (km, vm)):
                assert np.array_equal(x, y)
        finally:
            close_all([a, b, ta, tb])


def run_batch_vs_single(l2b, oracle, name, n, env, batched):
    """Sessions 0..n-1 (session 0 is the model's own context) against n twin sessions stepped one by one."""
    ck = payload(l2b, name)
    V, S, L = ck.vocab_size, ck.seq_len, ck.n_layers
    starts = [(61 * b) % (S // 2) for b in range(n)]
    steps = min(260, S - max(starts))
    toks = [stream(b, S, V) for b in range(n)]
    want = oracle_ref(l2b, oracle, name)[0]
    with l2b_env(env), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            for b in range(n):
                if starts[b]:
                    for t in (sess[b], twins[b]):
                        t.prefill(toks[b][:starts[b]], 0, want_logits=False)
            for i in range(steps):
                pos = [starts[b] + i for b in range(n)]
                tk = [toks[b][pos[b]] for b in range(n)]
                got = l2b.forward_batch(sess, tk, pos)
                k = sess[0].last_timing()[1]
                for b in range(n):
                    ref = twins[b].forward(tk[b], pos[b])
                    if batched:
                        assert rel_err(got[b], ref) <= 1e-6, (i, b, rel_err(got[b], ref))
                    else:
                        assert np.array_equal(got[b], ref), (i, b)
                step_launches = twins[0].last_timing()[1]
                assert k == (batch_launches(L, n) if batched else n * step_launches), (i, k)
                if starts[0] == 0 and i in want:
                    assert rel_err(got[0], want[i]) <= REL_TOL, (i, rel_err(got[0], want[i]))
                if i % 37 == 0 or i == steps - 1:
                    nxt = l2b.forward_argmax_batch(sess, tk, pos)       # the same step again: idempotent
                    assert nxt.tolist() == [int(np.argmax(g)) for g in got], i
            for b in range(n):
                for x, y in zip(caches(sess[b]), caches(twins[b])):
                    if batched:
                        assert np.max(np.abs(x - y)) <= 1e-6 * np.max(np.abs(y)), b
                    else:
                        assert np.array_equal(x, y), b
                assert np.array_equal(sess[b].state("logits"), got[b])
        finally:
            close_all(sess[1:] + twins)


BATCH_CASES = [("B", {}, True), ("S", {}, False), ("B", {"L2B_PREFILL_BATCH": "0"}, False)]


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7])
@pytest.mark.parametrize("name,env,batched", BATCH_CASES, ids=["B", "S", "B-prefill-batch0"])
def test_batch_equals_single_steps(l2b, oracle, name, env, batched, n):
    assert batched_prefill(MODELS[name][0], env) == batched
    run_batch_vs_single(l2b, oracle, name, n, env, batched)


@pytest.mark.parametrize("kind", ["tie", "neg", "last"])
def test_batch_argmax_edges(l2b, kind):
    """The crafted classifiers of test_device_argmax_edges on B, through the batched classifier: every
    vector's argmax key must give the first-index argmax of its logits (and the crafted row)."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    data, a = crafted(l2b, "B", kind)
    ck = shape_checkpoint(MODELS["B"][0], data)
    V, n = ck.vocab_size, 5
    toks = [stream(b, 24, V) for b in range(n)]
    signs = set()
    with l2b_env({}), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        try:
            for pos in range(24):
                tk, ps = [toks[b][pos] for b in range(n)], [pos] * n
                lg = l2b.forward_batch(sess, tk, ps)
                assert sess[0].last_timing()[1] == batch_launches(ck.n_layers, n)
                nxt = l2b.forward_argmax_batch(sess, tk, ps)
                for b in range(n):
                    best = int(np.argmax(lg[b]))
                    assert nxt[b] == best, (pos, b)
                    if kind == "tie":
                        assert best in (5, 6) and lg[b][5] == lg[b][V - 1] and lg[b][6] == lg[b][V - 2], (pos, b)
                    elif kind == "last":
                        assert best in (V - 1, V - 2), (pos, b)
                    elif np.all(lg[b] > 0) or np.all(lg[b] < 0):
                        signs.add(bool(lg[b][0] > 0))
                        assert best == (int(np.argmax(a)) if lg[b][0] > 0 else int(np.argmin(a))), (pos, b)
            if kind == "neg":
                assert signs == {True, False}, signs
        finally:
            close_all(sess[1:])


def test_batch_refusals_change_nothing(l2b):
    ck, cs = payload(l2b, "B"), payload(l2b, "S")
    V = ck.vocab_size
    with l2b_env({}), l2b.Transformer(ck) as m, l2b.Transformer(cs) as other:
        a, b = m.session(), m.session()
        try:
            l2b.forward_batch([a, b], [3, 4], [0, 0])
            l2b.forward_batch([a, b], [5, 6], [1, 1])
            other.forward(1, 0)
            before = [caches(t) for t in (m, a, b, other)]
            bad = [([a, a], [1, 2], [2, 2], -1),            # the same session twice
                   ([a, other], [1, 2], [2, 1], -1),        # sessions of two models
                   ([a, b], [1, 2], [2, 3], -7),            # b has 2 positions: pos 3 skips ahead
                   ([a, b], [1, V], [2, 2], -1),            # token out of range
                   ([b, a], [-1, 2], [2, 2], -1),
                   ([a, b], [1, 2], [2, ck.seq_len], -1)]   # past seq_len
            for sess, tk, ps, code in bad:
                for fn in (l2b.forward_batch, l2b.forward_argmax_batch):
                    with pytest.raises(l2b.L2BError) as e:
                        fn(sess, tk, ps)
                    assert e.value.status == code, (tk, ps, e.value)
            with pytest.raises(l2b.L2BError) as e:
                l2b.forward_batch([], [], [])
            assert e.value.status == -1
            for t, (k, v) in zip((m, a, b, other), before):
                kk, vv = caches(t)
                assert np.array_equal(k, kk) and np.array_equal(v, vv)
        finally:
            close_all([a, b])


def test_sessions_outlive_the_model(l2b):
    import torch
    ck = payload(l2b, "B")
    toks = teacher_tokens(12, ck.vocab_size)
    with l2b_env({}), l2b.Transformer(ck) as t:          # kernels loaded once, before the baseline
        l2b.forward_batch([t], [1], [0])
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    with l2b_env({}):
        m = l2b.Transformer(ck)
        a, b = m.session(), m.session()
        with l2b.Transformer(ck) as twin:
            for t in (a, b, twin):
                t.prefill(toks[:10], 0, want_logits=False)
            m.close()                                     # the weights must stay for a and b
            ref = twin.forward(toks[10], 10)
            assert np.array_equal(a.forward(toks[10], 10), ref)
            got = l2b.forward_batch([b, a], [toks[10], toks[11]], [10, 11])
            assert rel_err(got[0], ref) <= 1e-6
            assert rel_err(got[1], twin.forward(toks[11], 11)) <= 1e-6
        a.close()
        assert b.forward(toks[11], 11).shape == (ck.vocab_size,)
        b.close()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    assert abs(free1 - free0) <= 128 << 20, (free0, free1)


@pytest.mark.parametrize("name", ["pf-hid19840", "pf-hid19844"])
def test_batch_envelope(l2b, name):
    """One side of the batched budget each: inside it the batched step runs (1e-6), past it each
    session's own step (bit for bit)."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    shape, seed, batched = ENVELOPE[name][0], ENVELOPE[name][1], ENVELOPE[name][5]
    ck = shape_checkpoint(shape)
    ck.data = l2b.synth_checkpoint_host(ck, seed)
    V, n, steps = ck.vocab_size, 3, 12
    starts = [0, 5, 17]
    toks = [stream(b, ck.seq_len, V) for b in range(n)]
    with l2b_env({}), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            for b in range(1, n):
                for t in (sess[b], twins[b]):
                    t.prefill(toks[b][:starts[b]], 0, want_logits=False)
            for i in range(steps):
                pos = [starts[b] + i for b in range(n)]
                tk = [toks[b][pos[b]] for b in range(n)]
                got = l2b.forward_batch(sess, tk, pos)
                k = sess[0].last_timing()[1]
                for b in range(n):
                    ref = twins[b].forward(tk[b], pos[b])
                    if batched:
                        assert rel_err(got[b], ref) <= 1e-6, (i, b)
                    else:
                        assert np.array_equal(got[b], ref), (i, b)
                single = twins[0].last_timing()[1]
                assert k == (batch_launches(ck.n_layers, n) if batched else n * single), (i, k)
        finally:
            close_all(sess[1:] + twins)


@pytest.mark.slow
def test_llama2_7b_four_sessions(l2b):
    """llama2-7B at full depth: one model (26.4 GB) and 4 sessions (2.15 GB of KV cache each) fit where 4
    contexts (4 copies of the weights) would not.  8 batched steps == the same positions re-run one by
    one on the same sessions, within 1e-6."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint((4096, 11008, 32, 32, 32, -32000, 2048))
    V, n = ck.vocab_size, 4
    starts = [0, 61, 122, 183]
    toks = [stream(b, 200, V) for b in range(n)]
    with l2b_env({}), l2b.Transformer(ck, synthetic_seed=7) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        try:
            for b in range(1, n):
                sess[b].prefill(toks[b][:starts[b]], 0, want_logits=False)
            got = []
            for i in range(8):
                pos = [starts[b] + i for b in range(n)]
                got.append(l2b.forward_batch(sess, [toks[b][pos[b]] for b in range(n)], pos))
                assert sess[0].last_timing()[1] == batch_launches(32, n)
            for i in range(8):
                for b in range(n):
                    ref = sess[b].forward(toks[b][starts[b] + i], starts[b] + i)
                    assert rel_err(got[i][b], ref) <= 1e-6, (i, b, rel_err(got[i][b], ref))
        finally:
            close_all(sess[1:])
