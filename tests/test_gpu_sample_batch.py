"""GPU: the sampled step of several sessions in one call (l2b_forward_sample_batch).

Where l2b_forward_batch shares weight passes (pf_prepare in csrc/llama2_b200.cu), each group of up to 4
sessions runs the batched layers and the batched classifier, then sample_prep_batch_kernel: one CTA per
vector, in place on the group's logits rows, with the session's own temperature and top-p, writing the
session's own candidate list and count.  Its body is sample_prep_kernel's (sample_prep_row), so a row
holds exactly what the single kernel makes of the same logits.  Elsewhere each session runs
l2b_forward_sample's own step.  Session b samples with (T, p) = PARAMS[b % 4], so every batch of two or
more mixes a filtering session with one that does not filter.  The checks here:

  * equal to the pieces: the same step re-run with forward_batch (idempotent), each row through
    sample_prep (sample_prep_kernel on the host's copy), gives bit for bit the probabilities, candidates
    and count of forward_sample_batch; against twin sessions stepped with forward_sample, bit for bit on
    the fallback and within 1e-4 x max p on the batched path; the launch count shows which path ran;
    each session's state("logits") is its probabilities; session 0 against the oracle's float64 softmax;
  * the candidate overflow (n_cand = minus the host filter's count) next to a session that does not filter;
  * sampled generation with a seeded host draw equals per-session forward_sample loops, token for token;
  * refusals return their code and leave every cache unchanged;
  * both sides of the batched budget (test_gpu_envelope's pf-hid19840 / pf-hid19844), and llama2-7B at
    full depth with 4 sessions (slow).

Ledger: kernel or path -> a test that runs it
  sample_prep_batch_kernel, groups of 1-4 vectors, filtering and plain rows mixed
                                             test_sample_batch_equals_pieces[B-*], test_sample_batch_envelope[pf-hid19840],
                                             test_sample_batch_overflow[B]
  sample_prep_batch_kernel, candidate overflow
                                             test_sample_batch_overflow[B]
  fallback: each session's G_SAMPLE graph    test_sample_batch_equals_pieces[S-*], [B-prefill-batch0-*],
                                             test_sample_batch_generation[*], test_sample_batch_envelope[pf-hid19844],
                                             test_sample_batch_overflow[S]
  fallback: eager sample step (no graphs)    test_sample_batch_equals_pieces[S-no-graph-*]
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_envelope import ENVELOPE
from test_gpu_generate_batch import prefill_all
from test_gpu_sessions import batch_launches, caches, close_all, stream
from test_gpu_transformer import REL_TOL, rel_err
from test_gpu_variants import MODELS, batched_prefill, host_candidates, l2b_env, oracle_ref, payload, softmax64

pytestmark = pytest.mark.gpu

PARAMS = [(1.0, 0.9), (0.8, 0.0), (1.3, 1.0), (0.5, 0.95)]   # (temperature, top_p) of session b % 4
CAP = 8192                                                    # candidates the device keeps per session


def params(n):
    return [PARAMS[b % 4][0] for b in range(n)], [PARAMS[b % 4][1] for b in range(n)]


def filters(p):
    return p != 0.0 and p != 1.0                              # :1009


def prep(l2b, logits, temperature, top_p, cap=CAP):
    """sample_prep_kernel on one logits row, in l2b_forward_sample's terms: (probs, candidates or None,
    n_cand), n_cand 0 without the filter and minus the count when more than min(cap, 8192) passed."""
    probs, cand, k = l2b.sample_prep(logits, temperature, top_p, cand_cap=cap)
    if not filters(top_p):
        return probs, None, 0
    if k > min(cap, CAP):
        return probs, None, -k
    return probs, cand, k


def assert_same(got, want, where):
    (p, c, k), (wp, wc, wk) = got, want
    assert np.array_equal(p, wp), where
    assert k == wk, (where, k, wk)
    assert (c is None) == (wc is None), where
    if c is not None:
        assert np.array_equal(c["prob"], wc["prob"]) and np.array_equal(c["index"], wc["index"]), where


def check_step(l2b, sess, twins, tk, pos, temp, top_p, batched, cap=CAP):
    """One forward_sample_batch step against its pieces and against twin sessions; returns its output."""
    n, L = len(sess), sess[0].ck.n_layers
    probs, cands, counts = l2b.forward_sample_batch(sess, tk, pos, temp, top_p, cand_cap=cap)
    launches = sess[0].last_timing()[1]
    for b in range(n):
        assert np.array_equal(sess[b].state("logits"), probs[b]), b
    lg = l2b.forward_batch(sess, tk, pos)                     # the same step again: idempotent
    for b in range(n):
        got = (probs[b], cands[b], counts[b])
        assert_same(got, prep(l2b, lg[b], temp[b], top_p[b], cap), b)
        ref = twins[b].forward_sample(tk[b], pos[b], temp[b], top_p[b], cand_cap=cap, with_count=True)
        if batched:
            assert np.max(np.abs(probs[b] - ref[0])) <= 1e-4 * np.max(ref[0]), b
        else:
            assert_same(got, ref, b)
    single = twins[0].last_timing()[1]                        # one l2b_forward_sample step
    assert launches == (batch_launches(L, n) + (n + 3) // 4 if batched else n * single), launches
    return probs, cands, counts


SAMPLE_CASES = [("B", {}, True), ("S", {}, False), ("B", {"L2B_PREFILL_BATCH": "0"}, False),
                ("S", {"L2B_NO_GRAPH": "1"}, False)]


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7])
@pytest.mark.parametrize("name,env,batched", SAMPLE_CASES, ids=["B", "S", "B-prefill-batch0", "S-no-graph"])
def test_sample_batch_equals_pieces(l2b, oracle, name, env, batched, n):
    assert batched_prefill(MODELS[name][0], env) == batched
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    starts = [(61 * b) % (S // 2) for b in range(n)]
    steps = min(260, S - max(starts))
    toks = [stream(b, S, V) for b in range(n)]
    want = oracle_ref(l2b, oracle, name)[0]
    temp, top_p = params(n)
    with l2b_env(env), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            prefill_all((sess, twins), toks, starts)
            for i in range(steps):
                pos = [starts[b] + i for b in range(n)]
                probs, _, _ = check_step(l2b, sess, twins, [toks[b][pos[b]] for b in range(n)], pos, temp, top_p, batched)
                if i in want:                                  # session 0 starts at 0: the oracle's stream
                    exact = softmax64(want[i].astype(np.float64) / temp[0])
                    assert rel_err(probs[0], exact) <= REL_TOL, (i, rel_err(probs[0], exact))
        finally:
            close_all(sess[1:] + twins)


@pytest.mark.parametrize("name", ["B", "S"])
def test_sample_batch_overflow(l2b, name):
    """A flat distribution (T = 4, p = 0.999) passes far more than 16 candidates: with cand_cap = 16 the
    filtering sessions report minus the host filter's count, and the session that does not filter 0."""
    ck = payload(l2b, name)
    V, n, cap = ck.vocab_size, 3, 16
    temp, top_p = [4.0, 1.0, 4.0], [0.999, 1.0, 0.999]
    toks = [stream(b, 8, V) for b in range(n)]
    batched = batched_prefill(MODELS[name][0], {})
    with l2b_env({}), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            for pos in range(4):
                tk = [toks[b][pos] for b in range(n)]
                probs, cands, counts = check_step(l2b, sess, twins, tk, [pos] * n, temp, top_p, batched, cap=cap)
                assert counts[1] == 0 and cands[1] is None
                for b in (0, 2):
                    keep = host_candidates(probs[b], top_p[b])
                    assert keep.size > cap and counts[b] == -keep.size and cands[b] is None, (pos, b)
        finally:
            close_all(sess[1:] + twins)


def draw(rng, probs, cand, n_cand, top_p):
    """The host's part of sampling: top-p (:770-797) over the candidates, or over probs when more passed
    than the device returned, or the CDF walk over every probability without the filter (:728-741)."""
    r = rng.random()
    if n_cand == 0:
        idx, pr = np.arange(probs.size), probs
    else:
        if n_cand < 0:
            idx = host_candidates(probs, top_p)
            pr = probs[idx]
        else:
            idx, pr = cand["index"], cand["prob"]
        order = np.argsort(-pr, kind="stable")
        idx, pr = idx[order], pr[order]
        last = min(int(np.searchsorted(np.cumsum(pr, dtype=np.float64), top_p, side="right")), idx.size - 1)
        idx, pr = idx[:last + 1], pr[:last + 1]
    cdf = np.cumsum(pr, dtype=np.float64)
    return int(idx[min(int(np.searchsorted(cdf, r * cdf[-1], side="right")), idx.size - 1)])


@pytest.mark.parametrize("name,env", [("S", {}), ("B", {"L2B_PREFILL_BATCH": "0"})], ids=["S", "B-prefill-batch0"])
def test_sample_batch_generation(l2b, name, env):
    """3 sessions sample 64 positions each through forward_sample_batch, each with its own seeded host
    draw, the drawn token fed back: the same streams as per-session forward_sample loops."""
    assert not batched_prefill(MODELS[name][0], env)
    ck = payload(l2b, name)
    n, steps = 3, 64
    temp, top_p = params(n)
    with l2b_env(env), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            rngs = [np.random.default_rng(1000 + b) for b in range(n)]
            tok, got = [1] * n, [[] for _ in range(n)]
            for pos in range(steps):
                probs, cands, counts = l2b.forward_sample_batch(sess, tok, [pos] * n, temp, top_p)
                tok = [draw(rngs[b], probs[b], cands[b], counts[b], top_p[b]) for b in range(n)]
                for b in range(n):
                    got[b].append(tok[b])
            for b in range(n):
                rng, t, want = np.random.default_rng(1000 + b), 1, []
                for pos in range(steps):
                    probs, cand, k = twins[b].forward_sample(t, pos, temp[b], top_p[b], with_count=True)
                    t = draw(rng, probs, cand, k, top_p[b])
                    want.append(t)
                assert got[b] == want, b
            assert len(set(sum(got, []))) > n                  # the draws are not degenerate
        finally:
            close_all(sess[1:] + twins)


def test_sample_batch_refusals_change_nothing(l2b):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck, cs = payload(l2b, "B"), payload(l2b, "S")
    nan = float("nan")
    with l2b_env({}), l2b.Transformer(ck) as m, l2b.Transformer(cs) as other:
        a, b = m.session(), m.session()
        try:
            for t in (a, b):
                t.prefill([3, 4], 0, want_logits=False)
            other.forward(1, 0)
            before = [caches(t) for t in (m, a, b, other)]
            ok_t, ok_p = [1.0, 0.8], [0.9, 0.0]
            bad = [([a, a], [2, 2], ok_t, ok_p, CAP, -1),              # the same session twice
                   ([a, other], [2, 1], ok_t, ok_p, CAP, -1),          # sessions of two models
                   ([a, b], [2, 3], ok_t, ok_p, CAP, -7),              # b has 2 positions: pos 3 skips ahead
                   ([a, b], [2, 2], [1.0, 0.0], ok_p, CAP, -1),        # temperature 0 (greedy is argmax_batch's)
                   ([a, b], [2, 2], [-1.0, 1.0], ok_p, CAP, -1),
                   ([a, b], [2, 2], [1.0, nan], ok_p, CAP, -1),
                   ([a, b], [2, 2], ok_t, [-0.1, 0.9], CAP, -1),       # top_p outside [0, 1]
                   ([a, b], [2, 2], ok_t, [0.9, 1.1], CAP, -1),
                   ([a, b], [2, 2], ok_t, [nan, 0.9], CAP, -1),
                   ([a, b], [2, 2], ok_t, ok_p, 0, -1)]                # a filtering session, cand_cap 0
            for sess, ps, temp, top_p, cap, code in bad:
                with pytest.raises(l2b.L2BError) as e:
                    l2b.forward_sample_batch(sess, [1, 2], ps, temp, top_p, cand_cap=cap)
                assert e.value.status == code, (ps, temp, top_p, cap, e.value)
            lib = l2b.load_library()
            hs = (C.c_void_p * 2)(a.h.value, b.h.value)
            tk, ps = (C.c_int32 * 2)(1, 2), (C.c_int32 * 2)(2, 2)
            temp, top_p = (C.c_float * 2)(1.0, 0.8), (C.c_float * 2)(0.9, 0.0)
            cand, n_cand = (l2b.binding.L2BProbIndex * 16)(), (C.c_int32 * 2)()
            fs = lib.l2b_forward_sample_batch
            assert fs(hs, 2, tk, ps, temp, top_p, None, None, 8, n_cand) == -1    # filtering, no candidates
            assert fs(hs, 2, tk, ps, temp, top_p, None, cand, 8, None) == -1      # filtering, no count
            assert fs(hs, 2, tk, ps, None, top_p, None, cand, 8, n_cand) == -1    # NULL temperature
            assert fs(hs, 2, tk, ps, temp, None, None, cand, 8, n_cand) == -1     # NULL top_p
            for t, (k, v) in zip((m, a, b, other), before):
                kk, vv = caches(t)
                assert np.array_equal(k, kk) and np.array_equal(v, vv)
            # no session filters: cand, n_cand and host_probs may all be NULL
            plain = (C.c_float * 2)(1.0, 0.0)
            assert fs(hs, 2, tk, ps, temp, plain, None, None, 0, None) == 0
            probs, _, counts = l2b.forward_sample_batch([a, b], [1, 2], [2, 2], [1.0, 0.8], [1.0, 0.0])
            assert counts.tolist() == [0, 0]
            assert np.array_equal(a.state("logits"), probs[0]) and np.array_equal(b.state("logits"), probs[1])
        finally:
            close_all([a, b])

    # a 1-entry vocabulary has no top-p cutoff (:761 divides by n - 1)
    v1 = shape_checkpoint(ENVELOPE["vocab1"][0])
    v1.data = l2b.synth_checkpoint_host(v1, ENVELOPE["vocab1"][1])
    with l2b_env({}), l2b.Transformer(v1) as m:
        s = m.session()
        try:
            m.forward(0, 0)
            before = [caches(t) for t in (m, s)]
            with pytest.raises(l2b.L2BError) as e:
                l2b.forward_sample_batch([m, s], [0, 0], [1, 0], [1.0, 1.0], [0.9, 0.0])
            assert e.value.status == -1
            for t, (k, v) in zip((m, s), before):
                kk, vv = caches(t)
                assert np.array_equal(k, kk) and np.array_equal(v, vv)
        finally:
            s.close()


@pytest.mark.parametrize("name", ["pf-hid19840", "pf-hid19844"])
def test_sample_batch_envelope(l2b, name):
    """One side of the batched budget each: inside it the batched sampler runs, past it each session's
    own sample step."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    shape, seed, batched = ENVELOPE[name][0], ENVELOPE[name][1], ENVELOPE[name][5]
    ck = shape_checkpoint(shape)
    ck.data = l2b.synth_checkpoint_host(ck, seed)
    V, n, steps = ck.vocab_size, 3, 12
    starts = [0, 5, 17]
    toks = [stream(b, ck.seq_len, V) for b in range(n)]
    temp, top_p = params(n)
    with l2b_env({}), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            prefill_all((sess, twins), toks, starts)
            for i in range(steps):
                pos = [starts[b] + i for b in range(n)]
                check_step(l2b, sess, twins, [toks[b][pos[b]] for b in range(n)], pos, temp, top_p, batched)
        finally:
            close_all(sess[1:] + twins)


@pytest.mark.slow
def test_llama2_7b_four_sessions_sampled(l2b):
    """llama2-7B at full depth (26.4 GB of weights, 2.15 GB of KV cache per session), 4 sessions and 4
    twins: 4 sampled batched steps, each equal to its pieces bit for bit and within 1e-4 x max p of
    forward_sample."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint((4096, 11008, 32, 32, 32, -32000, 2048))
    V, n = ck.vocab_size, 4
    starts = [0, 61, 122, 183]
    toks = [stream(b, 200, V) for b in range(n)]
    temp, top_p = params(n)
    with l2b_env({}), l2b.Transformer(ck, synthetic_seed=7) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            prefill_all((sess, twins), toks, starts)
            for i in range(4):
                pos = [starts[b] + i for b in range(n)]
                check_step(l2b, sess, twins, [toks[b][pos[b]] for b in range(n)], pos, temp, top_p, True)
        finally:
            close_all(sess[1:] + twins)
