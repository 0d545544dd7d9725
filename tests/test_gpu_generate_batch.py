"""GPU: the greedy loop of several sessions on the device (l2b_generate_argmax_batch).

Where l2b_forward_batch shares weight passes (pf_prepare in csrc/llama2_b200.cu), the call enqueues
every step of every group of 4 sessions at once: batch_advance_kernel turns each vector's argmax key
(or its forced token) into the session's next token on the device, a stopped session's done flag keeps
its qkv kernel from appending KV rows, and once every session has stopped the queued kernels return at
once (CTL_DONE).  Elsewhere each session replays its own l2b_generate_argmax graph on its own stream.
The checks here:

  * fallback (S, and B with L2B_PREFILL_BATCH=0): tokens, n_done and both KV caches equal
    l2b_generate_argmax on twin sessions bit for bit, and the launches are the sum of the twins';
  * the stories15M-shaped golden stream on 3 sessions, and the BOS stop at position 19 of
    oracle_lib.bos_stop_payload on 2 sessions, with and without stop_on_bos;
  * batched path (B): tokens and KV caches equal, bit for bit, a host loop of l2b_forward_argmax_batch
    over twin sessions fed the same tokens in the same groups (the same kernels with the same arguments),
    and the launches are n_steps x (batched step + one advance per group);
  * stops on the batched path: a forced BOS stops one session while the others run on, its cache past
    the stop is untouched; a session started 3 positions before seq_len runs 3 steps; when every session
    has stopped, the rest of the call costs a fraction of the steps it skipped (device time);
  * refusals return their code and change no cache; l2b_generate_argmax refuses an out-of-range forced
    token too;
  * llama2-7B at full depth with 4 sessions (slow).
"""
import json
import hashlib
import os

import numpy as np
import pytest

from test_gpu_sessions import batch_launches, caches, close_all, stream
from test_gpu_transformer import GOLDEN
from test_gpu_variants import MODELS, batched_prefill, l2b_env, payload

pytestmark = pytest.mark.gpu


def staggered(n, seq_len):
    return [(61 * b) % (seq_len // 2) for b in range(n)]


def prompts(n, n_steps, starts, toks):
    """forced[b]: session b's next plen_b teacher tokens (plen_b differs per session; fewer where the
    stream ends), then -1."""
    forced = np.full((n, n_steps), -1, np.int32)
    for b in range(n):
        seg = toks[b][starts[b] + 1:starts[b] + 1 + min(n_steps, 2 + 3 * b)]
        forced[b, :len(seg)] = seg
    return forced


def prefill_all(groups, toks, starts):
    for b, s in enumerate(starts):
        if s:
            for ts in groups:
                ts[b].prefill(toks[b][:s], 0, want_logits=False)


def host_loop(l2b, twins, tokens, starts, n_steps, forced, stop_on_bos):
    """What l2b_generate_argmax_batch does on the batched path, one l2b_forward_argmax_batch per step:
    a stopped session stays in its group (its position held at seq_len - 1), fed its last token.
    Returns each session's tokens and its caches as they were when it stopped."""
    n, S = len(twins), twins[0].ck.seq_len
    limit = [min(n_steps, S - p) for p in starts]
    tok, outs, live, snaps = list(tokens), [[] for _ in range(n)], [True] * n, [None] * n
    for s in range(max(limit)):
        nxt = l2b.forward_argmax_batch(twins, tok, [min(p + s, S - 1) for p in starts])
        for b in range(n):
            if not live[b]:
                continue
            t = int(forced[b][s]) if forced is not None and forced[b][s] >= 0 else int(nxt[b])
            outs[b].append(t)
            tok[b] = t
            if (stop_on_bos and t == 1) or s + 1 == limit[b]:
                live[b], snaps[b] = False, caches(twins[b])
    return outs, snaps


@pytest.mark.parametrize("n", [1, 2, 3, 5])
@pytest.mark.parametrize("name,env", [("S", {}), ("B", {"L2B_PREFILL_BATCH": "0"})], ids=["S", "B-prefill-batch0"])
def test_fallback_equals_generate_argmax(l2b, name, env, n):
    assert not batched_prefill(MODELS[name][0], env)
    ck = payload(l2b, name)
    V, S, n_steps = ck.vocab_size, ck.seq_len, 40
    starts = staggered(n, S)
    toks = [stream(b, S, V) for b in range(n)]
    forced = prompts(n, n_steps, starts, toks)
    first = [toks[b][starts[b]] for b in range(n)]
    with l2b_env(env), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            prefill_all((sess, twins), toks, starts)
            got = l2b.generate_argmax_batch(sess, first, starts, n_steps, forced=forced, stop_on_bos=True)
            launches = sess[0].last_timing()[1]
            want, want_launches = [], 0
            for b in range(n):
                want.append(twins[b].generate_argmax(first[b], starts[b], n_steps, forced=forced[b], stop_on_bos=True))
                want_launches += twins[b].last_timing()[1]
            for b in range(n):
                assert got[b].tolist() == want[b].tolist(), b
                for x, y in zip(caches(sess[b]), caches(twins[b])):
                    assert np.array_equal(x, y), b
            assert launches == want_launches, (launches, want_launches)
        finally:
            close_all(sess[1:] + twins)


def test_golden_stream_and_bos_stop(l2b, oracle, stories15m):
    with open(os.path.join(GOLDEN, "stories15M_t0_tokens.json")) as f:
        gold = json.load(f)
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    want = gold["tokens"] + ([gold["terminator"]] if gold["terminator"] is not None else [])
    with l2b.Transformer(ck) as m:
        sess = [m, m.session(), m.session()]
        try:
            got = l2b.generate_argmax_batch(sess, [1, 1, 1], [0, 0, 0], 256, stop_on_bos=True)
            for out in got:
                assert out.tolist() == want and len(out) == gold["forward_calls"]
                toks = out[:len(gold["tokens"])]
                assert hashlib.sha256(np.array(toks, "<u4").tobytes()).hexdigest() == gold["sha256_le_u32"]
        finally:
            close_all(sess[1:])

    from llama2_zig_b200.checkpoint import shape_checkpoint
    k = oracle.BOS_STOP_POS
    ck = shape_checkpoint(oracle.BOS_STOP_SHAPE)
    ck.data = oracle.bos_stop_payload()
    with l2b.Transformer(ck) as m:
        sess = [m, m.session()]
        try:
            got = l2b.generate_argmax_batch(sess, [1, 1], [0, 0], 256, stop_on_bos=True)
            for out in got:
                assert len(out) == k + 1 and out[k] == 1 and 1 not in out[:k].tolist()
            run_on = l2b.generate_argmax_batch(sess, [1, 1], [0, 0], 256, stop_on_bos=False)
            for out, stopped in zip(run_on, got):
                assert len(out) == 256 and out[:k + 1].tolist() == stopped.tolist()
        finally:
            close_all(sess[1:])


def check_device_vs_host(l2b, sess, twins, first, starts, n_steps, forced, stop_on_bos):
    got = l2b.generate_argmax_batch(sess, first, starts, n_steps, forced=forced, stop_on_bos=stop_on_bos)
    want, snaps = host_loop(l2b, twins, first, starts, n_steps, forced, stop_on_bos)
    for b in range(len(sess)):
        assert got[b].tolist() == want[b], b
        for x, y in zip(caches(sess[b]), snaps[b]):
            assert np.array_equal(x, y), b
    return got


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7])
def test_batched_equals_host_loop(l2b, n):
    assert batched_prefill(MODELS["B"][0], {})
    ck = payload(l2b, "B")
    V, S, L, n_steps = ck.vocab_size, ck.seq_len, ck.n_layers, 40
    starts = staggered(n, S)
    toks = [stream(b, S, V) for b in range(n)]
    forced = prompts(n, n_steps, starts, toks)
    first = [toks[b][starts[b]] for b in range(n)]
    with l2b_env({}), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            prefill_all((sess, twins), toks, starts)
            got = check_device_vs_host(l2b, sess, twins, first, starts, n_steps, forced, True)
            assert all(len(g) == n_steps for g in got)
            groups = (n + 3) // 4
            assert sess[0].last_timing()[1] == n_steps * (batch_launches(L, n) + groups)
        finally:
            close_all(sess[1:] + twins)


def test_batched_stops(l2b):
    ck = payload(l2b, "B")
    V, S, n, n_steps = ck.vocab_size, ck.seq_len, 5, 30
    starts = [0, 61, 122, 183, S - 3]
    toks = [stream(b, S, V) for b in range(n)]
    forced = prompts(n, n_steps, starts, toks)
    forced[1, :7] = toks[1][starts[1] + 1:starts[1] + 8]
    forced[1, 6] = 1                                             # session 1 emits BOS at step 6
    first = [toks[b][starts[b]] for b in range(n)]
    with l2b_env({}), l2b.Transformer(ck) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            prefill_all((sess, twins), toks, starts)
            k1, v1 = caches(sess[1])
            got = check_device_vs_host(l2b, sess, twins, first, starts, n_steps, forced, True)
            assert len(got[1]) == 7 and got[1][6] == 1
            assert len(got[4]) == 3
            assert [len(got[b]) for b in (0, 2, 3)] == [n_steps] * 3
            kv = ck.dim * ck.n_kv_heads // ck.n_heads
            stop = starts[1] + 7
            for before, after in zip((k1, v1), caches(sess[1])):
                before, after = before.reshape(ck.n_layers, S, kv), after.reshape(ck.n_layers, S, kv)
                assert np.array_equal(before[:, stop:], after[:, stop:])

            # every session stops at step 2: the rest of a 200-step call must cost a fraction of 200 steps
            for s in sess:
                s.reset()
            twos = np.full((n, 200), -1, np.int32)
            twos[:, 2] = 1
            l2b.generate_argmax_batch(sess, [5] * n, [0] * n, 200, forced=twos, stop_on_bos=True)
            got = l2b.generate_argmax_batch(sess, [5] * n, [0] * n, 200, forced=twos, stop_on_bos=True)
            stopped_ms = sess[0].last_timing()[0]
            assert [len(g) for g in got] == [3] * n
            l2b.generate_argmax_batch(sess, [5] * n, [0] * n, 200, stop_on_bos=False)
            full_ms = sess[0].last_timing()[0]
            assert stopped_ms < 0.6 * full_ms, (stopped_ms, full_ms)
        finally:
            close_all(sess[1:] + twins)


def test_refusals_change_nothing(l2b):
    import ctypes as C
    ck, cs = payload(l2b, "B"), payload(l2b, "S")
    V = ck.vocab_size
    with l2b_env({}), l2b.Transformer(ck) as m, l2b.Transformer(cs) as other:
        a, b = m.session(), m.session()
        try:
            for t in (a, b):
                t.prefill([3, 4], 0, want_logits=False)
            other.forward(1, 0)
            before = [caches(t) for t in (m, a, b, other)]
            ok = np.full((2, 4), -1, np.int32)
            bad_forced = ok.copy()
            bad_forced[1, 3] = V
            low_forced = ok.copy()
            low_forced[0, 0] = -2
            bad = [([a, a], [1, 2], [2, 2], 4, ok, -1),              # the same session twice
                   ([a, other], [1, 2], [2, 1], 4, ok, -1),          # sessions of two models
                   ([a, b], [1, 2], [2, 3], 4, ok, -7),              # b has 2 positions: pos 3 skips ahead
                   ([a, b], [1, V], [2, 2], 4, ok, -1),              # token out of range
                   ([a, b], [1, 2], [2, 2], 4, bad_forced, -1),      # forced token out of range
                   ([a, b], [1, 2], [2, 2], 4, low_forced, -1),      # forced token below -1
                   ([a, b], [1, 2], [2, 2], -1, None, -1)]           # n_steps < 0
            for sess, tk, ps, n_steps, forced, code in bad:
                with pytest.raises(l2b.L2BError) as e:
                    l2b.generate_argmax_batch(sess, tk, ps, n_steps, forced=forced)
                assert e.value.status == code, (tk, ps, n_steps, e.value)
            lib = l2b.load_library()
            hs = (C.c_void_p * 2)(a.h.value, b.h.value)
            tk, ps = (C.c_int32 * 2)(1, 2), (C.c_int32 * 2)(2, 2)
            out, done = (C.c_int32 * 8)(), (C.c_int32 * 2)()
            assert lib.l2b_generate_argmax_batch(hs, 2, tk, ps, 4, None, 1, None, done) == -1
            assert lib.l2b_generate_argmax_batch(hs, 2, tk, ps, 4, None, 1, out, None) == -1
            # the same check on the single-context loop
            for f in ([1, 2, V, 3], [1, -2, -1, -1]):
                with pytest.raises(l2b.L2BError) as e:
                    a.generate_argmax(1, 2, 4, forced=np.array(f, np.int32))
                assert e.value.status == -1
            # n_steps == 0 runs nothing
            assert [len(g) for g in l2b.generate_argmax_batch([a, b], [1, 2], [2, 2], 0)] == [0, 0]
            for t, (k, v) in zip((m, a, b, other), before):
                kk, vv = caches(t)
                assert np.array_equal(k, kk) and np.array_equal(v, vv)
        finally:
            close_all([a, b])


@pytest.mark.slow
def test_llama2_7b_four_sessions_device_loop(l2b):
    """llama2-7B at full depth, 4 sessions from starts 0/61/122/183 (and 4 twins): 16 steps of the device
    loop, a 4-token forced prompt each then free-running, equal the host loop bit for bit."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint((4096, 11008, 32, 32, 32, -32000, 2048))
    V, n, n_steps = ck.vocab_size, 4, 16
    starts = [0, 61, 122, 183]
    toks = [stream(b, 220, V) for b in range(n)]
    forced = np.full((n, n_steps), -1, np.int32)
    for b in range(n):
        forced[b, :4] = toks[b][starts[b] + 1:starts[b] + 5]
    first = [toks[b][starts[b]] for b in range(n)]
    with l2b_env({}), l2b.Transformer(ck, synthetic_seed=7) as m:
        sess = [m] + [m.session() for _ in range(n - 1)]
        twins = [m.session() for _ in range(n)]
        try:
            prefill_all((sess, twins), toks, starts)
            got = check_device_vs_host(l2b, sess, twins, first, starts, n_steps, forced, True)
            assert all(len(g) == n_steps for g in got)
        finally:
            close_all(sess[1:] + twins)
