"""GPU: prompt chunks and decode steps of several sessions in one call (l2b_forward_ragged /
l2b_forward_argmax_ragged / l2b_forward_sample_ragged).

Session i runs its run of n_tokens[i] tokens at pos0[i] ..; the output is its last position's.  Where
l2b_prefill batches (pf_prepare in csrc/llama2_b200.cu), the runs' positions, concatenated in session
order, go 4 per pass over the weights through the batched step's kernels; a run may straddle passes,
and a pass holding no run's last position skips the classifier.  Elsewhere each session runs l2b_prefill
of all but its last token and then its own single step.  The claim under test is that a position's
arithmetic on the batched kernels depends on nothing else in its pass (not its slot, not the pass's
vector count), so a ragged call is its pieces bit for bit and a prompt gives the same bits however it
is cut into chunks.  The checks here:

  * pieces: each run's KV rows equal l2b_prefill of the run, its logits and x equal l2b_prefill of all
    but its last token followed by l2b_forward_batch (batched) or l2b_forward (fallback) of the last one,
    all bit for bit; within 1e-6 of l2b_forward position by position on the batched path; the runs
    straddle passes, mix a decode vector with another session's prompt, end exactly at seq_len and start
    at staggered positions; the launch count follows the per-pass formula;
  * chunk invariance: a 300-token prompt fed in irregular chunks across 256 (its queries change split
    count mid-prompt), next to other sessions' decode steps, leaves the cache of one l2b_prefill;
  * all ones: every n_tokens == 1 is the *_batch call bit for bit, with its launch count, in all modes;
  * argmax == the first-index np.argmax of the logits mode; the sampled mode == l2b_op_sample_prep of the
    logits mode's rows bit for bit, candidates included (a straddling run ends with its last row's), and
    the candidate overflow rule;
  * the fallback (S, B with L2B_PREFILL_BATCH=0), the golden stories15M stream, both sides of the batched
    budget (pf-hid19840 / pf-hid19844), refusals that change no cache, and llama2-7B (slow).

Ledger: path -> a test that runs it
  batched runs, passes with and without a run's last vector   test_ragged_equals_pieces[B-*]
  last rows moved to the front of the batch logits before the sampler
                                                              test_ragged_equals_pieces[B-mixed], [B-long-first]
  fallback: l2b_prefill + each session's own step graph      test_ragged_equals_pieces[S-*], [B-prefill-batch0-*],
                                                              test_ragged_envelope[pf-hid19844]
"""
import json
import os

import numpy as np
import pytest

from test_gpu_envelope import ENVELOPE
from test_gpu_sample_batch import PARAMS, assert_same, prep
from test_gpu_sessions import caches, close_all, stream
from test_gpu_transformer import rel_err
from test_gpu_variants import MODELS, batched_prefill, host_candidates, l2b_env, payload

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def ragged_launches(n_layers, lens, sample=False):
    """Kernels of one batched ragged call: the runs' vectors in passes of 4; per pass and layer qkv,
    attention, wo, w13 and one w2 per pair, then the classifier (and the sampler) when the pass holds
    some run's last vector."""
    ends, total = set(), 0
    for k in lens:
        total += k
        ends.add(total - 1)
    count = 0
    for g in range(0, total, 4):
        nb = min(4, total - g)
        count += n_layers * (4 + (nb + 1) // 2)
        if any(g <= e < g + nb for e in ends):
            count += 2 if sample else 1
    return count


def sample_params(n):
    """(temperature, top_p) per session: the first two filter, so a straddling second run filters."""
    ps = [PARAMS[(b + 3) % 4] for b in range(n)]
    return [p[0] for p in ps], [p[1] for p in ps]


def prefill_to(groups, toks, starts):
    for b, s in enumerate(starts):
        if s:
            for ts in groups:
                ts[b].prefill(toks[b][:s], 0, want_logits=False)


def check_pieces(l2b, ck, lens, starts, env):
    """One ragged call of each mode on sessions at `starts` against its pieces on twin sessions."""
    batched = batched_prefill(ck.shape_tuple, env)
    V, L, n = ck.vocab_size, ck.n_layers, len(lens)
    toks = [stream(b, ck.seq_len, V) for b in range(n)]
    runs = [toks[b][starts[b]:starts[b] + lens[b]] for b in range(n)]
    assert [len(r) for r in runs] == lens
    temp, top_p = sample_params(n)
    with l2b_env(env), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        pf = [m.session() for _ in range(n)]          # l2b_prefill of the whole run
        st = [m.session() for _ in range(n)]          # all but the last token, then the last one's step
        fw = [m.session() for _ in range(n)] if batched else []   # l2b_forward position by position
        try:
            prefill_to([sess, pf, st] + ([fw] if batched else []), toks, starts)
            got = l2b.forward_ragged(sess, runs, starts)
            launches = sess[0].last_timing()[1]
            want_launches = 0
            for b, (r, p0) in enumerate(zip(runs, starts)):
                last = p0 + len(r) - 1
                pf[b].prefill(r, p0, want_logits=False)
                if len(r) > 1:
                    st[b].prefill(r[:-1], p0, want_logits=False)
                    want_launches += st[b].last_timing()[1]
                ref = l2b.forward_batch([st[b]], [r[-1]], [last])[0] if batched else st[b].forward(r[-1], last)
                want_launches += st[b].last_timing()[1]
                assert np.array_equal(got[b], ref), b
                assert np.array_equal(sess[b].state("logits"), got[b]), b
                assert np.array_equal(sess[b].state("x"), st[b].state("x")), b
                for x, y, z in zip(caches(sess[b]), caches(pf[b]), caches(st[b])):
                    assert np.array_equal(x, y) and np.array_equal(x, z), b
                if batched:
                    for j, t in enumerate(r):
                        lg = fw[b].forward(t, p0 + j)
                    assert rel_err(got[b], lg) <= 1e-6, (b, rel_err(got[b], lg))
                    for x, y in zip(caches(sess[b]), caches(fw[b])):
                        assert np.max(np.abs(x - y)) <= 1e-6 * np.max(np.abs(y)), b
            assert launches == (ragged_launches(L, lens) if batched else want_launches), (launches, want_launches)

            # the same runs again (idempotent) in the other two modes
            nxt = l2b.forward_argmax_ragged(sess, runs, starts)
            assert nxt.tolist() == [int(np.argmax(g)) for g in got]
            if batched:
                assert sess[0].last_timing()[1] == ragged_launches(L, lens)
            probs, cands, counts = l2b.forward_sample_ragged(sess, runs, starts, temp, top_p)
            if batched:
                assert sess[0].last_timing()[1] == ragged_launches(L, lens, sample=True)
            for b in range(n):
                assert_same((probs[b], cands[b], counts[b]), prep(l2b, got[b], temp[b], top_p[b]), b)
                assert np.array_equal(sess[b].state("logits"), probs[b]), b
                for x, y in zip(caches(sess[b]), caches(pf[b])):
                    assert np.array_equal(x, y), b
        finally:
            close_all(sess[1:] + pf + st + fw)


def ragged_cases(seq_len):
    """name -> (run lengths, first positions): 'mixed' straddles passes (the second run spans two), puts a
    decode vector next to another session's prompt and ends a run at seq_len; 'long-first' has passes
    with no run's last vector; 'one-prompt' crosses the 256-position attention split inside the run."""
    return {"mixed": ([1, 7, 1, 3, 2], [0, 61, 122, seq_len - 3, 40]),
            "long-first": ([9, 1], [17, seq_len - 10]),
            "one-prompt": ([11], [250])}


PIECE_CASES = [("B", {}, True), ("S", {}, False), ("B", {"L2B_PREFILL_BATCH": "0"}, False)]


@pytest.mark.parametrize("case", ["mixed", "long-first", "one-prompt"])
@pytest.mark.parametrize("name,env,batched", PIECE_CASES, ids=["B", "S", "B-prefill-batch0"])
def test_ragged_equals_pieces(l2b, name, env, batched, case):
    assert batched_prefill(MODELS[name][0], env) == batched
    ck = payload(l2b, name)
    lens, starts = ragged_cases(ck.seq_len)[case]
    check_pieces(l2b, ck, lens, starts, env)


@pytest.mark.parametrize("name", ["pf-hid19840", "pf-hid19844"])
def test_ragged_envelope(l2b, name):
    """One side of the batched budget each: inside it the batched runs, past it each session's prefill
    and own step; bit for bit their pieces either way."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    shape, seed, batched = ENVELOPE[name][0], ENVELOPE[name][1], ENVELOPE[name][5]
    assert batched_prefill(shape, {}) == batched
    ck = shape_checkpoint(shape)
    ck.data = l2b.synth_checkpoint_host(ck, seed)
    check_pieces(l2b, ck, [1, 5, 2, 3], [0, 5, 17, ck.seq_len - 3], {})


def test_ragged_chunk_invariance(l2b):
    """A 300-token prompt in 14 irregular chunks, each next to two other sessions' decode steps (one of
    them crossing position 256 too): its cache equals one l2b_prefill of the prompt, and the decoders
    equal twins stepped alone with l2b_forward_batch, bit for bit."""
    ck = payload(l2b, "B")
    V, L = ck.vocab_size, ck.n_layers
    chunks = [3, 1, 6, 2, 11, 1, 40, 5, 90, 7, 100, 2, 17, 15]
    assert sum(chunks) == 300
    prompt = stream(9, 300, V)
    starts = [50, 250]
    toks = [stream(b, ck.seq_len, V) for b in range(2)]
    with l2b_env({}), l2b.Transformer(ck) as m:
        p, d0, d1 = m.session(), m.session(), m.session()
        whole, last, t0, t1 = m.session(), m.session(), m.session(), m.session()
        try:
            for d, t, s, tk in ((d0, t0, starts[0], toks[0]), (d1, t1, starts[1], toks[1])):
                for x in (d, t):
                    x.prefill(tk[:s], 0, want_logits=False)
            done = 0
            for i, c in enumerate(chunks):
                pos = [starts[0] + i, done, starts[1] + i]
                runs = [[toks[0][pos[0]]], prompt[done:done + c], [toks[1][pos[2]]]]
                got = l2b.forward_ragged([d0, p, d1], runs, pos)
                assert d0.last_timing()[1] == ragged_launches(L, [1, c, 1]), i
                assert np.array_equal(got[0], l2b.forward_batch([t0], runs[0], [pos[0]])[0]), i
                assert np.array_equal(got[2], l2b.forward_batch([t1], runs[2], [pos[2]])[0]), i
                done += c
            whole.prefill(prompt, 0, want_logits=False)
            for x, y in zip(caches(p), caches(whole)):
                assert np.array_equal(x, y)
            last.prefill(prompt[:-1], 0, want_logits=False)
            assert np.array_equal(got[1], l2b.forward_batch([last], [prompt[-1]], [299])[0])
            for d, t in ((d0, t0), (d1, t1)):
                for x, y in zip(caches(d), caches(t)):
                    assert np.array_equal(x, y)
        finally:
            close_all([p, d0, d1, whole, last, t0, t1])


@pytest.mark.parametrize("name,batched", [("B", True), ("S", False)])
def test_ragged_all_ones_is_the_batch_call(l2b, name, batched):
    """Every run of length 1: each mode equals its *_batch call on twin sessions bit for bit, with the
    same launch count."""
    assert batched_prefill(MODELS[name][0], {}) == batched
    ck = payload(l2b, name)
    V, S, n = ck.vocab_size, ck.seq_len, 6
    starts = [(61 * b) % (S // 2) for b in range(n)]
    toks = [stream(b, S, V) for b in range(n)]
    temp, top_p = sample_params(n)
    with l2b_env({}), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            prefill_to([sess, twins], toks, starts)
            for i in range(6):
                pos = [starts[b] + i for b in range(n)]
                tk = [toks[b][pos[b]] for b in range(n)]
                runs = [[t] for t in tk]
                got = l2b.forward_ragged(sess, runs, pos)
                k = sess[0].last_timing()[1]
                want = l2b.forward_batch(twins, tk, pos)
                assert np.array_equal(got, want) and k == twins[0].last_timing()[1], i
                got = l2b.forward_argmax_ragged(sess, runs, pos)
                k = sess[0].last_timing()[1]
                want = l2b.forward_argmax_batch(twins, tk, pos)
                assert np.array_equal(got, want) and k == twins[0].last_timing()[1], i
                got = l2b.forward_sample_ragged(sess, runs, pos, temp, top_p)
                k = sess[0].last_timing()[1]
                want = l2b.forward_sample_batch(twins, tk, pos, temp, top_p)
                assert k == twins[0].last_timing()[1], i
                for b in range(n):
                    assert_same((got[0][b], got[1][b], got[2][b]), (want[0][b], want[1][b], want[2][b]), (i, b))
            for b in range(n):
                for x, y in zip(caches(sess[b]), caches(twins[b])):
                    assert np.array_equal(x, y), b
        finally:
            close_all(sess[1:] + twins)


@pytest.mark.parametrize("name", ["B", "S"])
def test_ragged_sample_overflow(l2b, name):
    """A flat distribution (T = 4, p = 0.999) with cand_cap = 16: the filtering runs (one of them
    straddling a pass) report minus the host filter's count, the one that does not filter 0."""
    ck = payload(l2b, name)
    V, cap = ck.vocab_size, 16
    temp, top_p = [4.0, 1.0, 4.0], [0.999, 1.0, 0.999]
    lens = [3, 1, 6]
    toks = [stream(b, 8, V) for b in range(3)]
    runs = [toks[b][:lens[b]] for b in range(3)]
    with l2b_env({}), l2b.Transformer(ck) as m:
        sess = [m, m.session(), m.session()]
        try:
            probs, cands, counts = l2b.forward_sample_ragged(sess, runs, [0, 0, 0], temp, top_p, cand_cap=cap)
            lg = l2b.forward_ragged(sess, runs, [0, 0, 0])
            assert counts[1] == 0 and cands[1] is None
            for b in (0, 2):
                assert np.array_equal(probs[b], prep(l2b, lg[b], temp[b], top_p[b], cap)[0]), b
                keep = host_candidates(probs[b], top_p[b])
                assert keep.size > cap and counts[b] == -keep.size and cands[b] is None, b
        finally:
            close_all(sess[1:])


def test_ragged_golden_stream(l2b, stories15m):
    """The stories15M-shaped checkpoint (fallback path): a run of BOS and the first k golden tokens gives
    next == golden[k], for four sessions with different k in one call."""
    with open(os.path.join(GOLDEN, "stories15M_t0_tokens.json")) as f:
        gold = json.load(f)["tokens"]
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    ks = [0, 5, 17, 40]
    with l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(len(ks) - 1)]
        try:
            runs = [[1] + gold[:k] for k in ks]
            nxt = l2b.forward_argmax_ragged(sess, runs, [0] * len(ks))
            assert nxt.tolist() == [gold[k] for k in ks]
            # continuing: the next chunk of each stream from where its run ended
            runs = [gold[k:k + 3] for k in ks]
            nxt = l2b.forward_argmax_ragged(sess, runs, [k + 1 for k in ks])
            assert nxt.tolist() == [gold[k + 3] for k in ks]
        finally:
            close_all(sess[1:])


def test_ragged_refusals_change_nothing(l2b):
    import ctypes as C
    ck, cs = payload(l2b, "B"), payload(l2b, "S")
    V, S = ck.vocab_size, ck.seq_len
    with l2b_env({}), l2b.Transformer(ck) as m, l2b.Transformer(cs) as other:
        a, b = m.session(), m.session()
        try:
            l2b.forward_ragged([a, b], [[3, 4, 5], [6, 7]], [0, 0])
            other.forward(1, 0)
            before = [caches(t) for t in (m, a, b, other)]
            bad = [([a, a], [[1], [2]], [3, 3], -1),                  # the same session twice
                   ([a, other], [[1], [2]], [3, 1], -1),              # sessions of two models
                   ([a, b], [[1, 2], []], [3, 2], -1),                # n_tokens < 1
                   ([a, b], [[1, 2], [3, 4]], [3, S - 1], -1),        # runs past seq_len
                   ([a, b], [[1, V, 2], [3]], [3, 2], -1),            # a token out of range inside a run
                   ([a, b], [[1, 2], [3, -1]], [3, 2], -1),
                   ([a, b], [[1, 2], [3]], [-1, 2], -1),              # pos0 < 0
                   ([a, b], [[1, 2], [3]], [3, 3], -7)]               # b has 2 positions: pos0 3 skips ahead
            for sess, runs, pos0, code in bad:
                for fn in (l2b.forward_ragged, l2b.forward_argmax_ragged):
                    with pytest.raises(l2b.L2BError) as e:
                        fn(sess, runs, pos0)
                    assert e.value.status == code, (runs, pos0, e.value)
                with pytest.raises(l2b.L2BError) as e:
                    l2b.forward_sample_ragged(sess, runs, pos0, [1.0, 1.0], [0.9, 0.0])
                assert e.value.status == code, (runs, pos0, e.value)
            with pytest.raises(l2b.L2BError) as e:                   # the sample call's own checks
                l2b.forward_sample_ragged([a, b], [[1, 2], [3]], [3, 2], [1.0, 0.0], [0.9, 0.0])
            assert e.value.status == -1
            lib = l2b.load_library()
            hs = (C.c_void_p * 2)(a.h.value, b.h.value)
            lens, tk, ps = (C.c_int32 * 2)(2, 1), (C.c_int32 * 3)(1, 2, 3), (C.c_int32 * 2)(3, 2)
            nxt = (C.c_int32 * 2)()
            assert lib.l2b_forward_argmax_ragged(hs, 2, None, tk, ps, nxt) == -1     # NULL n_tokens
            assert lib.l2b_forward_argmax_ragged(hs, 2, lens, tk, None, nxt) == -1   # NULL pos0
            assert lib.l2b_forward_argmax_ragged(hs, 2, lens, None, ps, nxt) == -1   # NULL tokens
            assert lib.l2b_forward_argmax_ragged(hs, 2, lens, tk, ps, None) == -1    # NULL next
            for t, (k, v) in zip((m, a, b, other), before):
                kk, vv = caches(t)
                assert np.array_equal(k, kk) and np.array_equal(v, vv)
            # pos0 == the positions appended is accepted
            assert lib.l2b_forward_argmax_ragged(hs, 2, lens, tk, ps, nxt) == 0
        finally:
            close_all([a, b])


@pytest.mark.slow
def test_llama2_7b_admission(l2b):
    """llama2-7B at full depth: three sessions decode while a fourth admits a 61-token prompt in chunks
    that fill every pass (1, 5, 9, 13 and 33 tokens next to the 3 decode steps).  Each output equals the
    same position re-run on its session with l2b_forward_batch, and the prompt's cache equals l2b_prefill
    of the prompt re-run on it, bit for bit."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint((4096, 11008, 32, 32, 32, -32000, 2048))
    V = ck.vocab_size
    chunks = [1, 5, 9, 13, 33]
    starts = [0, 61, 122]
    toks = [stream(b, 200, V) for b in range(3)]
    prompt = stream(3, 61, V)
    with l2b_env({}), l2b.Transformer(ck, synthetic_seed=7) as m:
        dec = [m, m.session(), m.session()]
        p = m.session()
        try:
            for b in (1, 2):
                dec[b].prefill(toks[b][:starts[b]], 0, want_logits=False)
            got, done = [], 0
            for i, c in enumerate(chunks):
                pos = [starts[b] + i for b in range(3)] + [done]
                runs = [[toks[b][pos[b]]] for b in range(3)] + [prompt[done:done + c]]
                got.append(l2b.forward_ragged(dec + [p], runs, pos))
                assert m.last_timing()[1] == ragged_launches(32, [1, 1, 1, c])
                done += c
            kp = caches(p)
            p.prefill(prompt, 0, want_logits=False)
            for x, y in zip(kp, caches(p)):
                assert np.array_equal(x, y)
            assert np.array_equal(got[-1][3], l2b.forward_batch([p], [prompt[-1]], [60])[0])
            for i in range(len(chunks)):
                for b in range(3):
                    ref = l2b.forward_batch([dec[b]], [toks[b][starts[b] + i]], [starts[b] + i])[0]
                    assert np.array_equal(got[i][b], ref), (i, b)
        finally:
            close_all(dec[1:] + [p])
