"""GPU: greedy speculative decoding (l2b_verify_argmax_ragged, l2b_generate_speculative).

A verify run [t, d_1 .. d_m] runs m + 1 consecutive positions of a session and keeps the longest prefix of
drafts the model agrees with.  A position's arithmetic does not depend on its pass, so the tokens and KV rows
are those of the plain greedy loop, l2b_generate_argmax_batch of one session, bit for bit, whatever the
drafts.  Where l2b_forward_ragged shares weight passes (B) the vectors go 4 per pass and
verify_accept_kernel decides the runs after each pass's classifier; elsewhere (S, and B with
L2B_PREFILL_BATCH=0) each run is l2b_score's device loop of single decode steps.  The checks here:

  * verify == greedy stream: drafts taken from a twin's generate_argmax_batch stream with one corruption at
    every index c (c = m: none), m in {0, 1, 2, 3, 4, 7, 8} (1, 2 and 3 passes); n_accept == c, the emitted
    tokens, KV rows [0, p + c + 1) and the exact appended count p + c + 1, at p = 40, across the 256-position
    attention split and on a run that ends at seq_len - 1 (S, B, B without batching);
  * all-ones runs equal forward_argmax_batch; 3 sessions in one call, runs straddling passes, equal their own
    single-session calls;
  * the BOS stop: oracle_lib.bos_stop_payload (fallback) and a B payload whose classifier row 1 is scaled
    until the batched greedy stream emits BOS early (batched);
  * refusals change no cache and no appended count;
  * generate_speculative == generate_argmax_batch of a twin (tokens, KV rows, both appended counts) for
    k in {0, 1, 3, 4, 8} with the target's own model as draft (every proposal accepted: each round takes the
    catch-up path, and rounds == ceil(n / (k + 1)) on S), a model of another seed (acceptance near 0) and
    the target's weights with a perturbed final rmsnorm (some rounds accept all, some reject);
  * two calls equal one; n_steps cut mid-round; the golden stories15M stream with a draft; llama2-7B with a
    stories15M-shaped draft (slow); tensor parallel is refused.

Ledger: kernel or path -> a test that runs it
  verify_accept_kernel, 1 .. 3 passes, 1 .. 3 runs   test_verify_equals_greedy_stream[B], test_verify_three_sessions[B]
  verify_accept_kernel, BOS stop                      test_verify_bos_stop_batched
  verify_accept_kernel, early exit (CTL_DONE)         test_verify_equals_greedy_stream[B] (c < m with m >= 4)
  fallback: G_SCORE_LOOP per run                      test_verify_equals_greedy_stream[S], [B-prefill-batch0]
  generate_speculative, batched / fallback verify     test_speculative_equals_greedy[B-*], [S-*]
"""
import json
import os

import numpy as np
import pytest

from test_gpu_fork import appended_is, assert_rows, rows
from test_gpu_sessions import caches, close_all, stream
from test_gpu_variants import MODELS, batched_prefill, l2b_env, payload

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MS = (0, 1, 2, 3, 4, 7, 8)
KS = (0, 1, 3, 4, 8)
CASES = [("S", {}, False), ("B", {}, True), ("B", {"L2B_PREFILL_BATCH": "0"}, False)]
IDS = ["S", "B", "B-prefill-batch0"]


def greedy_stream(l2b, twin, toks, p0, n):
    """n greedy tokens from (toks[p0], p0) on twin, after a prefill of toks[:p0]."""
    twin.reset()
    if p0:
        twin.prefill(toks[:p0], 0, want_logits=False)
    g = l2b.generate_argmax_batch([twin], [toks[p0]], [p0], n, stop_on_bos=False)[0]
    assert len(g) == n
    return g


def drafts(g, m, c, vocab):
    """g[:m] with entry c replaced by another token (c == m: no corruption)."""
    d = [int(x) for x in g[:m]]
    if c < m:
        d[c] = (d[c] + 1) % vocab
    return d


@pytest.mark.parametrize("name,env,batched", CASES, ids=IDS)
def test_verify_equals_greedy_stream(l2b, name, env, batched):
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    assert batched_prefill(MODELS[name][0], env) == batched
    toks = stream(0, S, V)
    with l2b_env(env), l2b.Transformer(ck) as src:
        s, twin = src.session(), src.session()
        try:
            for p0 in (40, 252, S - 9):
                g = greedy_stream(l2b, twin, toks, p0, 9)
                src.reset()
                src.prefill(toks[:p0], 0, want_logits=False)
                for m in MS:
                    for c in range(m + 1):
                        l2b.fork(src, [s], p0)
                        got, acc = l2b.verify_argmax_ragged([s], [[toks[p0]] + drafts(g, m, c, V)], [p0])
                        where = (p0, m, c)
                        assert acc.tolist() == [c], where
                        assert got[0].tolist() == g[:c + 1].tolist(), where
                        assert_rows(rows(s, p0 + c + 1), rows(twin, p0 + c + 1), where)
                        if p0 + c + 1 < S - 1:            # appended_is steps at p0 + c + 1
                            appended_is(l2b, s, p0 + c + 1, toks[0])
        finally:
            close_all([s, twin])


@pytest.mark.parametrize("name,env,batched", CASES, ids=IDS)
def test_verify_all_ones_is_the_batch_call(l2b, name, env, batched):
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    starts = [0, 17, 255, 3, 100]
    toks = [stream(b, S, V) for b in range(5)]
    with l2b_env(env), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(4)]
        twins = [m.session() for _ in range(5)]
        try:
            for b, p in enumerate(starts):
                for t in (sess[b], twins[b]):
                    if p:
                        t.prefill(toks[b][:p], 0, want_logits=False)
            last = [toks[b][p] for b, p in enumerate(starts)]
            got, acc = l2b.verify_argmax_ragged(sess, [[t] for t in last], starts)
            want = l2b.forward_argmax_batch(twins, last, starts)
            assert acc.tolist() == [0] * 5
            assert [int(x[0]) for x in got] == want.tolist()
            for b, p in enumerate(starts):
                assert_rows(rows(sess[b], p + 1), rows(twins[b], p + 1), b)
        finally:
            close_all(sess[1:] + twins)


@pytest.mark.parametrize("name,env,batched", CASES, ids=IDS)
def test_verify_three_sessions(l2b, name, env, batched):
    """Runs of 3, 6 and 2 positions (11 vectors: passes of 4, 4 and 3), the first with its second draft
    corrupted, in one call, equal each session's own call."""
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    starts, lens, corrupt = [30, 250, 7], [3, 6, 2], [1, 5, 1]
    toks = [stream(b, S, V) for b in range(3)]
    with l2b_env(env), l2b.Transformer(ck) as m:
        sess = [m.session() for _ in range(3)]
        solo = [m.session() for _ in range(3)]
        twin = m.session()
        try:
            runs = []
            for b in range(3):
                g = greedy_stream(l2b, twin, toks[b], starts[b], lens[b])
                runs.append([toks[b][starts[b]]] + drafts(g, lens[b] - 1, corrupt[b], V))
                for t in (sess[b], solo[b]):
                    t.prefill(toks[b][:starts[b]], 0, want_logits=False)
            got, acc = l2b.verify_argmax_ragged(sess, runs, starts)
            assert acc.tolist() == [1, 5, 1]
            for b in range(3):
                g1, a1 = l2b.verify_argmax_ragged([solo[b]], [runs[b]], [starts[b]])
                assert a1.tolist() == [acc[b]] and g1[0].tolist() == got[b].tolist(), b
                end = starts[b] + acc[b] + 1
                assert_rows(rows(sess[b], end), rows(solo[b], end), b)
                appended_is(l2b, sess[b], end, toks[b][0])
        finally:
            close_all(sess + solo + [twin])


def check_bos_verify(l2b, m, g, kb):
    """g: the greedy stream from (1, 0) with its first BOS at g[kb].  A run of 8 correct drafts over it stops
    at the BOS with stop_on_bos and accepts all 8 without."""
    p0 = max(0, kb - 2)
    run = [1 if p0 == 0 else int(g[p0 - 1])] + [int(x) for x in g[p0:p0 + 8]]
    for stop, want in ((True, kb - p0), (False, 8)):
        s = m.session()
        try:
            if p0:
                s.prefill([1] + [int(x) for x in g[:p0 - 1]], 0, want_logits=False)
            got, acc = l2b.verify_argmax_ragged([s], [run], [p0], stop_on_bos=stop)
            assert acc.tolist() == [want], (stop, kb)
            assert got[0].tolist() == g[p0:p0 + want + 1].tolist()
        finally:
            s.close()


def test_verify_bos_stop_fallback(l2b, oracle):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint(oracle.BOS_STOP_SHAPE)
    ck.data = oracle.bos_stop_payload()
    with l2b.Transformer(ck) as m:
        g = m.generate_argmax(1, 0, 40, stop_on_bos=False)
        kb = oracle.BOS_STOP_POS
        assert g[kb] == 1 and 1 not in g[:kb].tolist()
        check_bos_verify(l2b, m, g, kb)


def test_verify_bos_stop_batched(l2b):
    """B with classifier row 1 (BOS) scaled by the first factor that makes the batched greedy stream from BOS
    emit BOS within 40 steps."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    base = payload(l2b, "B")
    dim, V = base.dim, base.vocab_size
    assert not base.shared_weights
    for f in (4.0, 16.0, 64.0):
        ck = shape_checkpoint(MODELS["B"][0])
        ck.data = base.data.copy()
        wcls = ck.data.size - V * dim
        ck.data[wcls + dim:wcls + 2 * dim] *= f
        with l2b_env({}), l2b.Transformer(ck) as m:
            g = l2b.generate_argmax_batch([m], [1], [0], 60, stop_on_bos=False)[0]
            if 1 not in g[:40].tolist():
                continue
            kb = g.tolist().index(1)
            assert l2b.generate_argmax_batch([m], [1], [0], 60, stop_on_bos=True)[0].tolist() == g[:kb + 1].tolist()
            check_bos_verify(l2b, m, g, kb)
            return
    pytest.fail("no scale of classifier row 1 made the batched greedy stream emit BOS")


def test_verify_refusals_change_nothing(l2b):
    import ctypes as C
    ck, cs = payload(l2b, "B"), payload(l2b, "S")
    V, S = ck.vocab_size, ck.seq_len
    toks = stream(0, 40, V)
    with l2b_env({}), l2b.Transformer(ck) as m, l2b.Transformer(cs) as other:
        a, b = m.session(), m.session()
        sess, count = [m, a, b, other], [20, 10, 5, 3]
        try:
            for t, k in zip(sess, count):
                t.prefill(toks[:k] if t is not other else [1, 2, 3], 0, want_logits=False)
            before = [caches(t) for t in sess]
            bad = [([a, a], [[1, 2], [3]], [10, 10], -1),            # the same session twice
                   ([a, other], [[1, 2], [3]], [10, 3], -1),         # sessions of two models
                   ([a, b], [[1, 2], [3]], [10, 6], -7),             # b has 5 positions: pos 6 skips ahead
                   ([a, b], [[1, V], [3]], [10, 5], -1),             # a draft out of range
                   ([a, b], [[1, 2], []], [10, 5], -1),              # an empty run
                   ([a, b], [[1] * 4, [3]], [S - 3, 5], -1)]         # a run past seq_len
            for ss, runs, pos, code in bad:
                with pytest.raises(l2b.L2BError) as e:
                    l2b.verify_argmax_ragged(ss, runs, pos)
                assert e.value.status == code, (runs, pos, e.value)
            lib = l2b.load_library()
            hs = (C.c_void_p * 2)(a.h.value, b.h.value)
            lens, tk, ps = (C.c_int32 * 2)(2, 1), (C.c_int32 * 3)(1, 2, 3), (C.c_int32 * 2)(10, 5)
            gr, acc = (C.c_int32 * 3)(), (C.c_int32 * 2)()
            assert lib.l2b_verify_argmax_ragged(hs, 2, lens, tk, ps, 0, None, acc) == -1
            assert lib.l2b_verify_argmax_ragged(hs, 2, lens, tk, ps, 0, gr, None) == -1
            for t, (k, v) in zip(sess, before):
                kk, vv = caches(t)
                assert np.array_equal(k, kk) and np.array_equal(v, vv)
            for t, k in zip(sess, count):
                appended_is(l2b, t, k, 1)
        finally:
            close_all([a, b])


# ---- generate_speculative -----------------------------------------------------------------------------

OTHER = 99                                        # seed of the unrelated draft


def rms_final_offset(ck):
    """Offset of rms_final in the checkpoint payload (src/main.zig:85-112)."""
    dim, hid, L, V = ck.dim, ck.hidden_dim, ck.n_layers, ck.vocab_size
    kvd = dim // ck.n_heads * ck.n_kv_heads
    return V * dim + 2 * L * dim + 2 * L * dim * dim + 2 * L * dim * kvd + 3 * L * dim * hid


def make_draft(l2b, kind, m, name):
    """(draft, owned contexts): a session of the target's model ("own"), a small model of the target's
    vocabulary and another seed ("other"), the target's weights with a perturbed final rmsnorm ("near")."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = payload(l2b, name)
    if kind == "own":
        d = m.session()
        return d, [d]
    if kind == "other":
        d = l2b.Transformer(shape_checkpoint((256, 688, 1, 4, 4, -ck.vocab_size, ck.seq_len)), synthetic_seed=OTHER)
        return d, [d]
    near = shape_checkpoint(MODELS[name][0])
    near.data = ck.data.copy()
    off = rms_final_offset(ck)
    rng = np.random.default_rng(5)
    near.data[off:off + ck.dim] *= (1.0 + 0.2 * rng.standard_normal(ck.dim)).astype(np.float32)
    d = l2b.Transformer(near)
    return d, [d]


SPEC_CASES = [(n, k) for n in ("S", "B") for k in ("own", "other", "near")]


@pytest.mark.parametrize("name,kind", SPEC_CASES, ids=[f"{n}-{k}" for n, k in SPEC_CASES])
def test_speculative_equals_greedy(l2b, name, kind):
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    p, n = 230, 50                                # crosses the 256-position attention split
    toks = stream(0, S, V)
    with l2b_env({}), l2b.Transformer(ck) as m:
        twin = m.session()
        draft, owned = make_draft(l2b, kind, m, name)
        try:
            twin.prefill(toks[:p], 0, want_logits=False)
            want = l2b.generate_argmax_batch([twin], [toks[p]], [p], n, stop_on_bos=True)[0]
            want_rows = rows(twin, p + len(want))
            for k in KS:
                m.reset()
                m.prefill(toks[:p], 0, want_logits=False)
                draft.reset()
                draft.prefill(toks[:p], 0, want_logits=False)
                got, rounds = m.generate_speculative(draft, toks[p], p, n, k)
                assert got.tolist() == want.tolist(), k
                end = p + len(got)
                assert_rows(rows(m, end), want_rows, k)
                if kind == "own" and name == "S":        # single steps everywhere: the draft agrees bit for bit
                    assert rounds == -(-len(got) // (k + 1)), (k, rounds)
                    assert_rows(rows(draft, end), want_rows, k)
                assert 1 <= rounds <= len(got)
                ms, launches = m.last_timing()
                assert ms > 0.0 and launches > 0
                appended_is(l2b, m, end, 1)
                appended_is(l2b, draft, end, 1)
        finally:
            close_all([twin] + owned)


@pytest.mark.parametrize("name", ["S", "B"])
def test_speculative_two_calls_and_cuts(l2b, name):
    """Two calls (25 + 35) equal one of 60 and the greedy stream; n_steps 1, 2 and 7 cut rounds of k = 4."""
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    p = 20
    toks = stream(1, S, V)
    with l2b_env({}), l2b.Transformer(ck) as m:
        twin, draft = m.session(), m.session()
        near, owned = make_draft(l2b, "near", m, name)
        try:
            twin.prefill(toks[:p], 0, want_logits=False)
            want = l2b.generate_argmax_batch([twin], [toks[p]], [p], 60, stop_on_bos=False)[0]
            for d in (draft, near):
                for t in (m, d):
                    t.reset()
                    t.prefill(toks[:p], 0, want_logits=False)
                a, _ = m.generate_speculative(d, toks[p], p, 25, 3, stop_on_bos=False)
                b, _ = m.generate_speculative(d, a[-1], p + 25, 35, 3, stop_on_bos=False)
                assert a.tolist() + b.tolist() == want.tolist()
                assert_rows(rows(m, p + 60), rows(twin, p + 60), "two calls")
                for n in (1, 2, 7):
                    for t in (m, d):
                        t.reset()
                        t.prefill(toks[:p], 0, want_logits=False)
                    got, _ = m.generate_speculative(d, toks[p], p, n, 4, stop_on_bos=False)
                    assert got.tolist() == want[:n].tolist(), n
                    appended_is(l2b, m, p + n, 1)
                    appended_is(l2b, d, p + n, 1)
            # the end of the context: at most seq_len - pos tokens, as generate_argmax
            for t in (m, draft):
                t.reset()
                t.prefill(toks[:S - 6], 0, want_logits=False)
            twin.reset()
            twin.prefill(toks[:S - 6], 0, want_logits=False)
            got, _ = m.generate_speculative(draft, toks[S - 6], S - 6, 50, 8, stop_on_bos=False)
            assert got.tolist() == l2b.generate_argmax_batch([twin], [toks[S - 6]], [S - 6], 50, stop_on_bos=False)[0].tolist()
            assert len(got) == 6
        finally:
            close_all([twin, draft] + owned)


def test_speculative_refusals_change_nothing(l2b):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = payload(l2b, "S")
    V, S = ck.vocab_size, ck.seq_len
    with l2b_env({}), l2b.Transformer(ck) as m, \
            l2b.Transformer(shape_checkpoint((64, 172, 1, 4, 4, -(V + 1), S)), synthetic_seed=3) as wide, \
            l2b.Transformer(shape_checkpoint((64, 172, 1, 4, 4, -V, S - 1)), synthetic_seed=3) as short:
        d = m.session()
        sess, count = [m, d, wide, short], [12, 6, 2, 2]
        try:
            for t, k in zip(sess, count):
                t.prefill(list(range(1, k + 1)), 0, want_logits=False)
            before = [caches(t) for t in sess]
            bad = [(m, 1, 5, 4, 3, -1),                      # the draft is the target
                   (d, 1, 5, 4, -1, -1),                     # k < 0
                   (d, 1, 5, 4, 33, -1),                     # k above L2B_SPECULATIVE_MAX_K
                   (d, 1, 5, -1, 3, -1),                     # n_steps < 0
                   (d, V, 5, 4, 3, -1),                      # token out of range
                   (d, 1, S, 4, 3, -1),                      # pos out of range
                   (wide, 1, 2, 4, 3, -1),                   # another vocabulary size
                   (short, 1, 2, 4, 3, -1),                  # a draft seq_len below the target's
                   (d, 1, 7, 4, 3, -7)]                      # the draft has 6 positions
            for dr, tok, pos, n, k, code in bad:
                with pytest.raises(l2b.L2BError) as e:
                    m.generate_speculative(dr, tok, pos, n, k)
                assert e.value.status == code, (tok, pos, n, k, e.value)
            lib = l2b.load_library()
            import ctypes as C
            out, done = (C.c_int32 * 4)(), C.c_int32()
            assert lib.l2b_generate_speculative(m.h, None, 1, 2, 4, 3, 1, out, C.byref(done), None) == -1
            assert lib.l2b_generate_speculative(m.h, d.h, 1, 2, 4, 3, 1, None, C.byref(done), None) == -1
            assert lib.l2b_generate_speculative(m.h, d.h, 1, 2, 4, 3, 1, out, None, None) == -1
            for t, (k, v) in zip(sess, before):
                kk, vv = caches(t)
                assert np.array_equal(k, kk) and np.array_equal(v, vv)
            for t, k in zip(sess, count):
                appended_is(l2b, t, k, 1)
        finally:
            d.close()


def test_speculative_golden_stream(l2b, stories15m):
    """The stories15M-shaped golden stream from BOS, with a stories15M-shaped draft of another seed."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    with open(os.path.join(GOLDEN, "stories15M_t0_tokens.json")) as f:
        gold = json.load(f)
    want = gold["tokens"] + ([gold["terminator"]] if gold["terminator"] is not None else [])
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    with l2b.Transformer(ck) as m, \
            l2b.Transformer(shape_checkpoint((288, 768, 6, 6, 6, 32000, 256)), synthetic_seed=11) as draft:
        for k in (1, 3):
            m.reset()
            draft.reset()
            got, rounds = m.generate_speculative(draft, 1, 0, 256, k, stop_on_bos=True)
            assert got.tolist() == want and len(got) == gold["forward_calls"], k
            assert rounds <= len(got)


@pytest.mark.slow
def test_llama2_7b_speculative(l2b):
    """llama2-7B at full depth with a stories15M-shaped draft (seq_len 2048): 64 tokens after an 8-token
    prompt equal the batched greedy stream of a twin session, tokens and KV rows."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint((4096, 11008, 32, 32, 32, -32000, 2048))
    prompt = stream(3, 9, ck.vocab_size)
    p = len(prompt) - 1
    with l2b_env({}), l2b.Transformer(ck, synthetic_seed=7) as m, \
            l2b.Transformer(shape_checkpoint((288, 768, 6, 6, 6, 32000, 2048)), synthetic_seed=10) as draft:
        twin = m.session()
        try:
            for t in (m, twin, draft):
                t.prefill(prompt[:-1], 0, want_logits=False)
            want = l2b.generate_argmax_batch([twin], [prompt[-1]], [p], 64, stop_on_bos=False)[0]
            got, rounds = m.generate_speculative(draft, prompt[-1], p, 64, 3, stop_on_bos=False)
            assert got.tolist() == want.tolist()
            assert_rows(rows(m, p + 64), rows(twin, p + 64), "7B")
            assert 16 <= rounds <= 64
        finally:
            twin.close()


def test_speculative_refuses_tensor_parallel(l2b):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from llama2_zig_b200.checkpoint import shape_checkpoint
    shape = (256, 688, 2, 8, 4, 512, 64)
    with l2b.Transformer(shape_checkpoint(shape), synthetic_seed=11, n_gpus=2) as grp, \
            l2b.Transformer(shape_checkpoint(shape), synthetic_seed=11) as one:
        grp.forward(1, 0)
        one.forward(1, 0)
        for t, d in ((grp, one), (one, grp)):
            with pytest.raises(l2b.L2BError) as e:
                t.generate_speculative(d, 1, 1, 4, 3)
            assert e.value.status == -2
        with pytest.raises(l2b.L2BError) as e:
            l2b.verify_argmax_ragged([grp], [[1, 2]], [1])
        assert e.value.status == -2
