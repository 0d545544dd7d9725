"""GPU: forking sessions from a shared prompt (l2b_fork, `fork`).

l2b_fork copies rows [0, n_pos) of a source session's key and value caches, in every layer, into each
destination session of the same model; each destination then has exactly n_pos positions appended and
its rows from n_pos on are not written.  kv_fork_kernel (csrc/l2b_device.cuh) reads each source float4
once and stores it to up to 8 destinations; more destinations take one launch per group of 8.  The claim
under test is that a fork is, bit for bit, the destination's own l2b_prefill of the same tokens: a batched
position's arithmetic does not depend on its pass, and the fallback prefill is single decode steps.  The
checks here:

  * fork == own prefill: at n_pos in {0, 1, 7, 255, 256, 257, N}, on destinations that held other rows,
    rows [0, n_pos) equal a twin's prefill, rows past n_pos are untouched, the source is unchanged (caches,
    x, logits, appended count), and forward + generate_argmax + score continue bit for bit like the twin;
    on S (latency kernels, GQA), B (batched path), hs20 (MQA, kv_loc 20), 110M and B without batching;
  * fork then step together: forward_argmax_batch and forward_sample_batch of the last prompt token on the
    source and 3 forks equal 4 sessions that each prefilled the prompt (B batched, S fallback);
  * 17 destinations take 3 launches; n_pos == 0 launches nothing and leaves nothing appended;
  * a fork shrinks a longer stream; refusals change no cache and no appended count;
  * the golden stories15M stream continues on a fork; llama2-7B (slow); tensor parallel is refused.

Ledger: kernel or path -> a test that runs it
  kv_fork_kernel, 1 .. 8 destinations per launch   test_fork_equals_own_prefill[*], test_fork_then_step_together[*]
  kv_fork_kernel, groups of 8, 8 and 1             test_fork_many_destinations
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

from test_gpu_sample_batch import assert_same, params
from test_gpu_sessions import caches, close_all, stream
from test_gpu_variants import MODELS, batched_prefill, l2b_env, payload

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N_SRC = 260                                       # source positions: the continuation stays inside seq_len 300
CONT = 1 + 20 + 11                                # forward, 20 generated steps, a 12-token score


def rows(t, n, lo=0):
    """(key, value) cache rows [lo, n) of every layer of session t, as (L, n - lo, kv_dim) arrays."""
    ck = t.ck
    kv = ck.dim * ck.n_kv_heads // ck.n_heads
    return [c.reshape(ck.n_layers, ck.seq_len, kv)[:, lo:n] for c in caches(t)]


def assert_rows(a, b, where):
    for x, y in zip(a, b):
        assert np.array_equal(x, y), where


def appended_is(l2b, t, k, tok):
    """Session t has exactly k positions appended: forward at k + 1 is refused (L2B_ERR_STATE), forward at k
    is accepted.  The accepted step appends position k; returns k + 1."""
    with pytest.raises(l2b.L2BError) as e:
        t.forward(tok, k + 1)
    assert e.value.status == -7, k
    t.forward(tok, k)
    return k + 1


def continuation(t, toks, n_pos):
    """forward at n_pos, a 20-step greedy loop from n_pos + 1, a score of 12 tokens from n_pos + 21."""
    lg = t.forward(toks[n_pos], n_pos)
    gen = t.generate_argmax(int(np.argmax(lg)), n_pos + 1, 20, stop_on_bos=False)
    lp, greedy = t.score(toks[n_pos + 21:n_pos + 33], n_pos + 21)
    return lg, gen, lp, greedy


FORK_CASES = [("S", {}), ("B", {}), ("hs20", {}), ("110M", {}), ("B", {"L2B_PREFILL_BATCH": "0"})]


@pytest.mark.parametrize("name,env", FORK_CASES, ids=["S", "B", "hs20", "110M", "B-prefill-batch0"])
def test_fork_equals_own_prefill(l2b, name, env):
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    assert N_SRC + CONT <= S
    assert batched_prefill(MODELS[name][0], env) == (name == "B" and not env)
    toks = stream(0, S, V)
    other = [stream(5 + b, S, V) for b in range(3)]
    held = [N_SRC + CONT + 8, 100, 3]             # what each destination holds before every fork
    with l2b_env(env), l2b.Transformer(ck) as m:
        dst = [m.session() for _ in range(3)]
        twin = m.session()
        try:
            m.prefill(toks[:N_SRC], 0, want_logits=False)
            src_state = [m.state(k) for k in ("key_cache", "value_cache", "x", "logits")]
            for n_pos in (0, 1, 7, 255, 256, 257, N_SRC):
                for d, o, h in zip(dst, other, held):
                    d.reset()
                    d.prefill(o[:h], 0, want_logits=False)
                before = [caches(d) for d in dst]
                l2b.fork(m, dst, n_pos)
                assert m.last_timing()[1] == (1 if n_pos else 0), n_pos
                for k, v in zip(("key_cache", "value_cache", "x", "logits"), src_state):
                    assert np.array_equal(m.state(k), v), (n_pos, k)
                twin.reset()
                if n_pos:
                    twin.prefill(toks[:n_pos], 0, want_logits=False)
                want_rows = rows(twin, n_pos)
                for b, d in enumerate(dst):
                    assert_rows(rows(d, n_pos), want_rows, (n_pos, b))
                    lo = [c.reshape(ck.n_layers, S, -1)[:, n_pos:] for c in before[b]]
                    assert_rows(rows(d, S, n_pos), lo, (n_pos, b))
                want = continuation(twin, toks, n_pos)
                assert len(want[1]) == 20
                end = n_pos + CONT
                for b, d in enumerate(dst):
                    got = continuation(d, toks, n_pos)
                    for x, y in zip(got, want):
                        assert np.array_equal(x, y), (n_pos, b)
                    assert_rows(rows(d, end), rows(twin, end), (n_pos, b))
            # the source's appended count is still N_SRC
            appended_is(l2b, m, N_SRC, toks[N_SRC])
        finally:
            close_all(dst + [twin])


@pytest.mark.parametrize("name", ["B", "S"])
def test_fork_then_step_together(l2b, name):
    """The source prefills prompt[:-1] and forks to 3 sessions; one 4-session step of the last prompt token
    equals 4 sessions that each prefilled prompt[:-1], in the argmax and the sampled batch call."""
    ck = payload(l2b, name)
    V, P = ck.vocab_size, 43
    prompt = stream(11, P, V)
    temp, top_p = params(4)
    with l2b_env({}), l2b.Transformer(ck) as m:
        forks = [m.session() for _ in range(3)]
        twins = [m.session() for _ in range(4)]
        try:
            m.prefill(prompt[:-1], 0, want_logits=False)
            l2b.fork(m, forks, P - 1)
            for t in twins:
                t.prefill(prompt[:-1], 0, want_logits=False)
            sess = [m] + forks
            last, pos = [prompt[-1]] * 4, [P - 1] * 4
            got = l2b.forward_argmax_batch(sess, last, pos)
            assert np.array_equal(got, l2b.forward_argmax_batch(twins, last, pos))
            got = l2b.forward_sample_batch(sess, last, pos, temp, top_p)
            want = l2b.forward_sample_batch(twins, last, pos, temp, top_p)
            for b in range(4):
                assert_same((got[0][b], got[1][b], got[2][b]), (want[0][b], want[1][b], want[2][b]), b)
                assert_rows(rows(sess[b], P), rows(twins[b], P), b)
        finally:
            close_all(forks + twins)


def test_fork_many_destinations(l2b):
    """17 destinations: ceil(17 / 8) = 3 launches and every destination's rows equal the source's; a fork
    at n_pos 0 launches nothing and leaves every destination with nothing appended."""
    ck = payload(l2b, "S")
    toks = stream(0, 120, ck.vocab_size)
    with l2b_env({}), l2b.Transformer(ck) as m:
        dst = [m.session() for _ in range(17)]
        try:
            m.prefill(toks[:100], 0, want_logits=False)
            for d in dst[::4]:
                d.prefill(toks[50:110], 0, want_logits=False)
            l2b.fork(m, dst, 100)
            ms, launches = m.last_timing()
            assert launches == 3 and ms > 0.0
            want = rows(m, 100)
            for b, d in enumerate(dst):
                assert_rows(rows(d, 100), want, b)
            l2b.fork(m, dst, 0)
            assert m.last_timing() == (0.0, 0)
            for d in dst:
                with pytest.raises(l2b.L2BError) as e:
                    d.forward(toks[0], 1)
                assert e.value.status == -7
        finally:
            close_all(dst)


def test_fork_shrinks_a_stream(l2b):
    """A destination that holds 300 positions, forked at 100, continues at 100 and not past it."""
    ck = payload(l2b, "S")
    V = ck.vocab_size
    toks, long = stream(0, 120, V), stream(3, 300, V)
    with l2b_env({}), l2b.Transformer(ck) as m:
        d, twin = m.session(), m.session()
        try:
            m.prefill(toks[:110], 0, want_logits=False)
            d.prefill(long, 0, want_logits=False)
            twin.prefill(toks[:100], 0, want_logits=False)
            l2b.fork(m, [d], 100)
            with pytest.raises(l2b.L2BError) as e:
                d.forward(toks[100], 101)
            assert e.value.status == -7
            assert np.array_equal(d.forward(toks[100], 100), twin.forward(toks[100], 100))
            assert_rows(rows(d, 101), rows(twin, 101), "rows")
        finally:
            close_all([d, twin])


def test_fork_refusals_change_nothing(l2b):
    ck = payload(l2b, "S")
    toks = stream(0, 80, ck.vocab_size)
    lib = l2b.load_library()
    with l2b_env({}), l2b.Transformer(ck) as m, l2b.Transformer(ck) as other:
        a, b = m.session(), m.session()
        sess = [m, a, b, other]
        try:
            count = [50, 30, 10, 5]
            for t, k in zip(sess, count):
                t.prefill(toks[:k], 0, want_logits=False)
            before = [caches(t) for t in sess]

            def unchanged(where):
                for i, t in enumerate(sess):
                    for x, y in zip(caches(t), before[i]):
                        assert np.array_equal(x, y), (where, i)
                for i, t in enumerate(sess):
                    count[i] = appended_is(l2b, t, count[i], toks[count[i]])
                    before[i] = caches(t)

            bad = [([a, m], 5, -1, "src among the destinations"),
                   ([a, a], 5, -1, "the same destination twice"),
                   ([a, other], 5, -1, "a session of another model"),
                   ([a, b], -1, -1, "n_pos < 0"),
                   ([a, b], None, -7, "n_pos past the source's appended count")]   # None: appended + 1
            for dsts, n_pos, code, what in bad:
                with pytest.raises(l2b.L2BError) as e:
                    l2b.fork(m, dsts, count[0] + 1 if n_pos is None else n_pos)
                assert e.value.status == code, (what, e.value)
                unchanged(what)
            hs = (C.c_void_p * 2)(a.h.value, None)
            assert lib.l2b_fork(m.h, 5, hs, 2) == -1                  # a NULL entry
            assert b"NULL" in lib.l2b_last_error(m.h)
            assert lib.l2b_fork(m.h, 5, None, 2) == -1                # NULL dst
            assert lib.l2b_fork(m.h, 5, hs, 0) == -1                  # n_dst < 1
            unchanged("NULL arguments")
            # n_pos == the source's appended count is accepted
            l2b.fork(m, [a, b], count[0])
            assert_rows(rows(a, count[0]), rows(m, count[0]), "a")
        finally:
            close_all([a, b])


def test_fork_golden_stream(l2b, stories15m):
    """The stories15M-shaped checkpoint: a fork at 100 of the greedy stream continues it exactly."""
    with open(os.path.join(GOLDEN, "stories15M_t0_tokens.json")) as f:
        gold = json.load(f)["tokens"]
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    with l2b.Transformer(ck) as m:
        d = m.session()
        try:
            assert m.generate_argmax(1, 0, 120, stop_on_bos=False).tolist() == gold[:120]
            l2b.fork(m, [d], 100)
            assert d.generate_argmax(gold[99], 100, 156, stop_on_bos=False).tolist() == gold[100:256]
        finally:
            d.close()


@pytest.mark.slow
def test_llama2_7b_fork(l2b):
    """llama2-7B at full depth: 3 forks of a 255-position prefill against 3 twins that prefilled it, and one
    4-session argmax step of the last prompt token, bit for bit."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint((4096, 11008, 32, 32, 32, -32000, 2048))
    P = 256
    prompt = stream(3, P, ck.vocab_size)
    with l2b_env({}), l2b.Transformer(ck, synthetic_seed=7) as m:
        forks = [m.session() for _ in range(3)]
        twins = [m.session() for _ in range(3)]
        try:
            m.prefill(prompt[:-1], 0, want_logits=False)
            l2b.fork(m, forks, P - 1)
            for t in twins:
                t.prefill(prompt[:-1], 0, want_logits=False)
            for b in range(3):
                assert_rows(rows(forks[b], P - 1), rows(twins[b], P - 1), b)
            last, pos = [prompt[-1]] * 4, [P - 1] * 4
            got = l2b.forward_argmax_batch([m] + forks, last, pos)
            want = l2b.forward_argmax_batch([m] + twins, last, pos)
            assert np.array_equal(got, want)
        finally:
            close_all(forks + twins)


def test_fork_refuses_tensor_parallel(l2b):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from llama2_zig_b200.checkpoint import shape_checkpoint
    shape = (256, 688, 2, 8, 4, 512, 64)
    with l2b.Transformer(shape_checkpoint(shape), synthetic_seed=11, n_gpus=2) as grp, \
            l2b.Transformer(shape_checkpoint(shape), synthetic_seed=11) as one:
        grp.forward(1, 0)
        with pytest.raises(l2b.L2BError) as e:
            l2b.fork(grp, [one], 1)
        assert e.value.status == -2
