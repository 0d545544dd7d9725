"""GPU: per-position log-probabilities of a known sequence (l2b_score, Transformer.score).

l2b_score runs tokens[i] at position pos0+i for i < n-1 and returns log softmax(logits)[tokens[i+1]] and
the first-index argmax of each position's logits.  Where l2b_prefill batches (pf_prepare in
csrc/llama2_b200.cu) it runs l2b_prefill's groups of 4 positions, each followed by the batched argmax
classifier and logprob_batch_kernel (one CTA per row); elsewhere the device loop G_SCORE_LOOP replays a
decode step with the argmax classifier, logprob_kernel and the forced-token advance.  The checks here:

  * the op (l2b_op_logprob, logprob_row on one row) against the float64 log-softmax, up to 1e6 entries;
  * the fallback equals its pieces bit for bit: a twin session stepped with l2b_forward + l2b_op_logprob
    and l2b_forward_argmax, and both KV caches;
  * the batched path: KV caches bit for bit those of l2b_prefill(tokens[:-1]), logprob within
    2e-6 x max|logit| + 1e-5 of the log-softmax of l2b_forward's logits, greedy equal to their argmax
    wherever the top two differ by more than the logits' own error; every partial last group;
  * the launch count shows which path ran;
  * the golden stories15M stream, against the oracle's logits;
  * boundaries (seq_len), continuation with l2b_forward, n_tokens == 1, and refusals that change nothing;
  * llama2-7B at full depth (slow).

Ledger: kernel or path -> a test that runs it
  logprob_batch_kernel, groups of 1-4 rows     test_score_batched[*], test_score_boundaries[B], test_llama2_7b_score
  logprob_batch_kernel, one row (the op)       test_op_logprob[*]
  logprob_kernel in the G_SCORE_LOOP graph     test_score_fallback_equals_pieces[S|B-prefill-batch0|W-*],
                                               test_score_golden_stream, test_score_boundaries[S]
  logprob_kernel, eager (no graphs)            test_score_fallback_equals_pieces[S-no-graph-*]
"""
import json
import os

import numpy as np
import pytest

from test_gpu_sessions import caches, stream
from test_gpu_variants import MODELS, batched_prefill, l2b_env, payload, prefill_launches

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def exact_lp(logits, target):
    """float64 log softmax(logits)[target] of float32 logits."""
    x = np.asarray(logits, dtype=np.float64)
    m = np.max(x)
    return (x[target] - m) - np.log(np.sum(np.exp(x - m)))


def lp_bound(exact):
    return 1e-5 + 1e-6 * abs(exact)                            # fp32 sum of the exponentials + one logf


# ---- the op ------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 2, 31, 32000, 32003, 1000000])
def test_op_logprob(l2b, n):
    rng = np.random.default_rng(n)
    rows = [rng.standard_normal(n).astype(np.float32) * np.float32(3)]
    spread = rng.uniform(-5e3, 5e3, n).astype(np.float32)       # a logit spread of 1e4
    rows.append(spread)
    tie = rng.standard_normal(n).astype(np.float32)
    tie[[0, n // 2, n - 1]] = np.float32(4.5)                   # repeated maxima, first and last included
    rows.append(tie)
    for row in rows:
        for t in sorted({0, n - 1, int(np.argmax(row)), n // 3}):
            got = l2b.logprob(row, t)
            want = exact_lp(row, t)
            assert abs(got - want) <= lp_bound(want), (n, t, got, want)
            if n == 1:
                assert got == 0.0


# ---- the fallback: bit for bit its pieces -------------------------------------------------------

def stepped(l2b, twin, toks, pos0):
    """The pieces of a score on a twin: l2b_forward + l2b_op_logprob and l2b_forward_argmax per position.
    Returns (logits per position, logprob, greedy)."""
    logits, lp, greedy = [], [], []
    for i in range(len(toks) - 1):
        lg = twin.forward(toks[i], pos0 + i)
        logits.append(lg)
        lp.append(l2b.logprob(lg, toks[i + 1]))
        greedy.append(twin.forward_argmax(toks[i], pos0 + i))   # re-running a position is idempotent
    return logits, np.array(lp, np.float32), np.array(greedy, np.int32)


FALLBACK = [("S", {}), ("S", {"L2B_NO_GRAPH": "1"}), ("B", {"L2B_PREFILL_BATCH": "0"}), ("W", {})]


@pytest.mark.parametrize("name,env", FALLBACK, ids=["S", "S-no-graph", "B-prefill-batch0", "W"])
def test_score_fallback_equals_pieces(l2b, name, env):
    assert not batched_prefill(MODELS[name][0], env)
    ck = payload(l2b, name)
    V = ck.vocab_size
    with l2b_env(env), l2b.Transformer(ck) as m:
        twin = m.session()
        try:
            for pos0 in (0, 17):
                for n_tokens in (2, 5, 40):
                    toks = stream(3, pos0 + n_tokens, V)
                    for t in (m, twin):
                        t.reset()
                        if pos0:
                            t.prefill(toks[:pos0], 0, want_logits=False)
                    lp, greedy = m.score(toks[pos0:], pos0)
                    _, launches = m.last_timing()
                    _, want_lp, want_greedy = stepped(l2b, twin, toks[pos0:], pos0)
                    assert lp.shape == (n_tokens - 1,) and greedy.shape == (n_tokens - 1,)
                    assert np.array_equal(lp, want_lp), (pos0, n_tokens)
                    assert np.array_equal(greedy, want_greedy), (pos0, n_tokens)
                    for a, b in zip(caches(m), caches(twin)):
                        assert np.array_equal(a, b), (pos0, n_tokens)
                    twin.forward(toks[pos0], pos0)
                    step = twin.last_timing()[1]                  # one l2b_forward step (G_LOGITS)
                    assert launches == (n_tokens - 1) * (step + 2), (launches, step)   # + logprob + advance
        finally:
            twin.close()


# ---- the batched path -------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 9, 258])
def test_score_batched(l2b, n):
    env = {}
    assert batched_prefill(MODELS["B"][0], env)
    ck = payload(l2b, "B")
    V = ck.vocab_size
    with l2b_env(env), l2b.Transformer(ck) as m:
        pf, fw = m.session(), m.session()
        try:
            for pos0 in (0, 17):
                toks = stream(5, pos0 + n + 1, V)
                for t in (m, pf, fw):
                    t.reset()
                    if pos0:
                        t.prefill(toks[:pos0], 0, want_logits=False)
                lp, greedy = m.score(toks[pos0:], pos0)
                _, launches = m.last_timing()
                pf.prefill(toks[pos0:-1], pos0, want_logits=False)
                assert launches == pf.last_timing()[1] + 2 * ((n + 3) // 4)          # + classifier, logprob per group
                assert pf.last_timing()[1] == prefill_launches(ck.shape_tuple, env, n, None)
                for a, b in zip(caches(m), caches(pf)):
                    assert np.array_equal(a, b), pos0
                for i in range(n):
                    lg = fw.forward(toks[pos0 + i], pos0 + i)
                    scale = float(np.max(np.abs(lg)))
                    want = exact_lp(lg, toks[pos0 + i + 1])
                    assert abs(lp[i] - want) <= 2e-6 * scale + 1e-5, (pos0, i, lp[i], want)
                    top2 = np.sort(lg)[-2:]
                    if top2[1] - top2[0] > 2e-6 * scale:
                        assert greedy[i] == int(np.argmax(lg)), (pos0, i)
        finally:
            pf.close()
            fw.close()


# ---- the golden stream ------------------------------------------------------------------------

def test_score_golden_stream(l2b, oracle, stories15m):
    """[BOS] + the greedy stream of the stories15M-shaped checkpoint: every greedy token is the stream's
    next one; over 64 positions logprob is within the logits' tolerance of the oracle's log-softmax."""
    with open(os.path.join(GOLDEN, "stories15M_t0_tokens.json")) as f:
        gold = json.load(f)
    toks = [1] + gold["tokens"] + ([gold["terminator"]] if gold["terminator"] is not None else [])
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    cfg, shared, data = oracle.read_checkpoint(stories15m)
    om = oracle.OracleModel(cfg, data, shared, W=8, kind="strict")
    try:
        with l2b.Transformer(ck) as t:
            lp, greedy = t.score(toks, 0)
        assert greedy.tolist() == toks[1:]
        for pos in range(min(64, len(toks) - 1)):
            lg = om.forward(toks[pos], pos)
            want = exact_lp(lg, toks[pos + 1])
            assert abs(lp[pos] - want) <= 2e-4 * np.max(np.abs(lg)) + 1e-5, (pos, lp[pos], want)
    finally:
        om.close()


# ---- boundaries, continuation, refusals ----------------------------------------------------------

@pytest.mark.parametrize("name", ["S", "B"])
def test_score_boundaries(l2b, name):
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    toks = stream(7, S + 2, V)
    with l2b_env({}), l2b.Transformer(ck) as m:
        twin = m.session()
        try:
            # continuation: the next l2b_forward after a score equals the same step on a prefilled twin
            lp, _ = m.score(toks[:41], 0)
            assert lp.shape == (40,) and np.all(np.isfinite(lp)) and np.all(lp <= 0)
            twin.prefill(toks[:40], 0, want_logits=False)
            assert np.array_equal(m.forward(toks[40], 40), twin.forward(toks[40], 40))
            # n_tokens == 1 runs nothing and writes nothing
            before = caches(m)
            lp1, g1 = m.score([toks[41]], 41)
            assert lp1.size == 0 and g1.size == 0 and m.last_timing() == (0.0, 0)
            for a, b in zip(before, caches(m)):
                assert np.array_equal(a, b)
            # the last position of the context is scored; one more is refused
            m.reset()
            lp, greedy = m.score(toks[:S + 1], 0)
            assert lp.shape == (S,) and np.all(np.isfinite(lp)) and greedy.min() >= 0 and greedy.max() < V
            with pytest.raises(l2b.L2BError) as e:
                m.score(toks[:S + 2], 0)
            assert e.value.status == -1
            with pytest.raises(l2b.L2BError) as e:
                m.score(toks[:3], S - 1)
            assert e.value.status == -1
        finally:
            twin.close()


@pytest.mark.parametrize("name", ["S", "B"])
def test_score_refusals_change_nothing(l2b, name):
    ck = payload(l2b, name)
    V = ck.vocab_size
    with l2b_env({}), l2b.Transformer(ck) as m:
        m.prefill([3, 4, 5], 0, want_logits=False)
        before = caches(m)
        bad = [([1, 2, -1], 0, -1),              # a token out of range, also the last (a target)
               ([1, V, 2], 0, -1),
               ([1, 2, 3], 4, -7),               # pos0 past the 3 positions appended
               ([1, 2, 3], -1, -1),
               ([], 0, -1)]                      # n_tokens < 1
        for toks, pos0, code in bad:
            with pytest.raises(l2b.L2BError) as e:
                m.score(toks, pos0)
            assert e.value.status == code, (toks, pos0, e.value)
        for a, b in zip(before, caches(m)):
            assert np.array_equal(a, b)
        lp, _ = m.score([5, 6, 7], 3)            # pos0 == the positions appended is accepted
        assert lp.shape == (2,)


# ---- llama2-7B -------------------------------------------------------------------------------------

@pytest.mark.slow
def test_llama2_7b_score(l2b):
    """llama2-7B at full depth (bench.py's synthetic weights, seed 7): 64 tokens scored from position 0 on
    the batched path, against a session stepped with l2b_forward, within the batched bar."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint((4096, 11008, 32, 32, 32, -32000, 2048))
    toks = stream(0, 64, ck.vocab_size)
    with l2b_env({}), l2b.Transformer(ck, synthetic_seed=7) as m:
        s = m.session()
        try:
            lp, greedy = m.score(toks, 0)
            assert m.last_timing()[1] > 0
            for i in range(63):
                lg = s.forward(toks[i], i)
                scale = float(np.max(np.abs(lg)))
                want = exact_lp(lg, toks[i + 1])
                assert abs(lp[i] - want) <= 2e-6 * scale + 1e-5, (i, lp[i], want)
                top2 = np.sort(lg)[-2:]
                if top2[1] - top2[0] > 2e-6 * scale:
                    assert greedy[i] == int(np.argmax(lg)), i
        finally:
            s.close()
