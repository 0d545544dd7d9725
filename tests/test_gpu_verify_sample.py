"""GPU: sampled speculative decoding (l2b_verify_sample_ragged, the host twin's
l2h_generate_speculative_sample).

l2b_verify_sample_ragged returns the device sampler preparation at every position of its runs.  A position's
arithmetic does not depend on its pass, so row v equals l2b_forward_sample_ragged of a run ending at v, bit for
bit.  The host walks those rows with its sampler and the same coins (uniform draws of l2h_seed's PRNG) as the
plain loop, so the sampled stream is the plain loop's whatever the draft.  The checks here:

  * per position: probabilities, candidates and counts equal forward_sample_ragged of a run ending there,
    for one run of 1 .. 9 positions (1 to 3 passes on B) and three sessions whose runs straddle passes, with
    per-session temperature and top-p, and with a candidate buffer too small (the -count rule); the appended
    counts follow max(appended, pos0 + n_tokens) (S, B, B without batching);
  * refusals, among them a total above the staging cap, change no cache and no appended count;
  * l2h_generate_speculative_sample equals the plain loop (forward_sample_batch of one session and the twin's
    sampler, same seed): tokens, n_done and the target's KV rows, for k in {0, 1, 3, 8}, T in {0.7, 1.0},
    top-p in {0, 0.9}, with and without the BOS stop, with the target's own model as draft (every round
    accepted on S), an unrelated model and the target with a perturbed final rmsnorm; two calls continue one
    stream; the seq_len limit; the stories15M checkpoint as target;
  * the demo CLI prints the same text with --draft as with --device-sampler.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_gpu_fork import appended_is, assert_rows, rows
from test_gpu_sessions import caches, close_all, stream
from test_gpu_speculative import make_draft
from test_gpu_variants import MODELS, batched_prefill, l2b_env, payload
from test_host_twin import tokenizer_path  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP = C.POINTER(C.c_float)
IP = C.POINTER(C.c_int32)
CASES = [("S", {}, False), ("B", {}, True), ("B", {"L2B_PREFILL_BATCH": "0"}, False)]
IDS = ["S", "B", "B-prefill-batch0"]


class PI(C.Structure):
    _fields_ = [("prob", C.c_float), ("index", C.c_int32)]


@pytest.fixture(scope="module")
def host(l2b):
    path = os.path.join(ROOT, "llama2.zig_b200", "lib", "libllama2_host.so")
    C.CDLL(l2b.lib_path(), mode=C.RTLD_GLOBAL)
    lib = C.CDLL(path)
    lib.l2h_seed.argtypes = [C.c_uint64]
    lib.l2h_sample.argtypes = [FP, C.c_int32]
    lib.l2h_sample_top_p.argtypes = [FP, C.c_int32, C.c_float, C.c_void_p]
    lib.l2h_sample_top_p_candidates.argtypes = [C.POINTER(PI), C.c_int32, C.c_float]
    cfg = C.POINTER(l2b.L2BConfig)
    lib.l2h_generate_speculative_sample.argtypes = [
        C.c_void_p, cfg, C.c_void_p, cfg, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
        C.c_float, C.c_float, C.c_int32, IP, IP, IP]
    return lib


def sample(host, probs, cand, n_cand, top_p):
    """The device-sampler loop's pick (l2h_generate): the twin's exported sampler on one step's output."""
    V = probs.size
    if top_p in (0.0, 1.0):
        return host.l2h_sample(probs.ctypes.data_as(FP), V)
    if n_cand > 0:
        arr = (PI * n_cand).from_buffer_copy(cand.tobytes())
        return host.l2h_sample_top_p_candidates(arr, n_cand, top_p)
    return host.l2h_sample_top_p(probs.ctypes.data_as(FP), V, top_p, (C.c_uint64 * V)())


def plain_stream(l2b, host, t, token, pos, n, temp, top_p, stop_on_bos, seed=None):
    """The reference: per token one forward_sample_batch of t (n = 1) and the twin's sampler."""
    if seed is not None:
        host.l2h_seed(seed)
    out = []
    for q in range(pos, min(pos + n, t.ck.seq_len)):
        probs, cands, nc = l2b.forward_sample_batch([t], [token], [q], [temp], [top_p])
        token = sample(host, probs[0], cands[0], int(nc[0]), top_p)
        out.append(token)
        if stop_on_bos and token == 1:
            break
    return out


def speculative(host, target, draft, token, pos, n, k, temp, top_p, stop_on_bos, seed=None):
    if seed is not None:
        host.l2h_seed(seed)
    out = np.full(max(n, 1), -1, dtype=np.int32)
    done, rounds = C.c_int32(-1), C.c_int32(-1)
    rc = host.l2h_generate_speculative_sample(target.h, C.byref(target.cfg), draft.h, C.byref(draft.cfg), token, pos,
                                              n, k, temp, top_p, 1 if stop_on_bos else 0,
                                              out.ctypes.data_as(IP), C.byref(done), C.byref(rounds))
    assert rc == 0, (rc, target.lib.l2b_last_error(target.h), target.lib.l2b_last_error(draft.h))
    return out[:done.value].tolist(), rounds.value


def assert_same_rows(got, want, where):
    probs, cands, nc = got
    wp, wc, wn = want
    assert np.array_equal(probs, wp), where
    assert nc == wn, where
    if wn > 0:
        assert np.array_equal(cands, wc), where
    else:
        assert cands is None, where


# ---- per-position exactness ---------------------------------------------------------------------------

@pytest.mark.parametrize("name,env,batched", CASES, ids=IDS)
def test_every_position_equals_the_ragged_call(l2b, name, env, batched):
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    assert batched_prefill(MODELS[name][0], env) == batched
    toks = stream(0, S, V)
    p0 = 250                                           # runs cross the 256-position attention split
    with l2b_env(env), l2b.Transformer(ck) as src:
        ss = [src.session() for _ in range(3)]
        twin = src.session()
        try:
            src.prefill(toks[:p0], 0, want_logits=False)
            settings = [(0.7, 0.9), (1.0, 0.0), (1.3, 0.5)]
            # one run of 1 .. 9 positions (1 to 3 passes), then three runs that straddle passes
            calls = [([m], [0]) for m in range(1, 10)] + [([3, 5, 2], [0, 1, 2]), ([1, 4, 6], [2, 0, 1])]
            overflowed = 0
            for lens, which in calls:
                sess = [ss[i] for i in which]
                runs = [toks[p0:p0 + m] for m in lens]
                temp = [settings[i][0] for i in which]
                top_p = [settings[i][1] for i in which]
                for cap in (8192, 3):                  # 3: fewer than pass, n_cand = -count
                    l2b.fork(src, sess, p0)
                    got = l2b.verify_sample_ragged(sess, runs, [p0] * len(sess), temp, top_p, cand_cap=cap)
                    v = 0
                    for i, run in enumerate(runs):
                        for j in range(len(run)):
                            l2b.fork(src, [twin], p0)
                            want = l2b.forward_sample_ragged([twin], [run[:j + 1]], [p0], [temp[i]], [top_p[i]],
                                                             cand_cap=cap)
                            where = (lens, i, j, cap)
                            assert_same_rows((got[0][v], got[1][v], got[2][v]), (want[0][0], want[1][0], want[2][0]),
                                             where)
                            overflowed += cap == 3 and got[2][v] < 0
                            v += 1
                        assert_rows(rows(sess[i], p0 + len(run)), rows(twin, p0 + len(run)), (lens, i))
                    for s, run in zip(sess, runs):
                        appended_is(l2b, s, p0 + len(run), 1)
            assert overflowed > 0                      # the -count rule was exercised
            # a session that already holds more positions keeps its count: max(appended, pos0 + n_tokens)
            l2b.fork(src, [ss[0]], p0)
            ss[0].prefill(toks[p0:p0 + 12], p0, want_logits=False)
            l2b.verify_sample_ragged([ss[0]], [toks[p0:p0 + 4]], [p0], [1.0], [0.9])
            appended_is(l2b, ss[0], p0 + 12, 1)
            # host_probs NULL and no filtering session: no probabilities, no candidate buffer needed
            lib = l2b.load_library()
            hs = (C.c_void_p * 1)(ss[1].h.value)
            lens = (C.c_int32 * 1)(3)
            tk = (C.c_int32 * 3)(*toks[p0:p0 + 3])
            pos = (C.c_int32 * 1)(p0)
            l2b.fork(src, [ss[1]], p0)
            assert lib.l2b_verify_sample_ragged(hs, 1, lens, tk, pos, (C.c_float * 1)(1.0), (C.c_float * 1)(0.0),
                                                None, None, 0, None) == 0
            l2b.fork(src, [twin], p0)
            l2b.forward_sample_ragged([twin], [toks[p0:p0 + 3]], [p0], [1.0], [0.0])
            assert_rows(rows(ss[1], p0 + 3), rows(twin, p0 + 3), "NULL outputs")
        finally:
            close_all(ss + [twin])


@pytest.mark.parametrize("name", ["S", "B"])
def test_refusals_change_nothing(l2b, name):
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    toks = stream(2, S, V)
    with l2b_env({}), l2b.Transformer(ck) as m:
        ss = [m] + [m.session() for _ in range(3)]
        try:
            P = S - 12
            for t in ss:
                t.prefill(toks[:P], 0, want_logits=False)
            before = [caches(t) for t in ss]
            per_pos = 4 * V + 8 * 8192
            cap = (64 << 20) // per_pos
            n_runs = cap // (S - 10) + 1              # enough runs of S - 10 positions to pass the cap
            assert n_runs <= len(ss) and n_runs * (S - 10) > max(cap, 33 * n_runs)
            big = [toks[:S - 10]] * n_runs
            bad = [(ss[:n_runs], big, [0] * n_runs, [1.0] * n_runs, [0.9] * n_runs, -1),   # above the staging cap
                   ([m], [[1, 2]], [5], [0.0], [0.9], -1),                  # temperature 0
                   ([m], [[1, 2]], [5], [1.0], [1.5], -1),                  # top_p above 1
                   ([m], [[1, V]], [5], [1.0], [0.9], -1),                  # token out of range
                   ([m], [toks[:13]], [P], [1.0], [0.9], -1),               # run past seq_len
                   ([m, m], [[1], [2]], [1, 2], [1.0, 1.0], [0.9, 0.9], -1)]   # the same session twice
            for sess, runs, pos0, temp, top_p, code in bad:
                with pytest.raises(l2b.L2BError) as e:
                    l2b.verify_sample_ragged(sess, runs, pos0, temp, top_p)
                assert e.value.status == code, (pos0, temp, top_p, e.value)
            fresh = m.session()
            try:
                with pytest.raises(l2b.L2BError) as e:                       # pos0 past the appended count
                    l2b.verify_sample_ragged([fresh], [[1, 2]], [3], [1.0], [0.9])
                assert e.value.status == -7
            finally:
                fresh.close()
            lib = l2b.load_library()                                          # a filtering session without candidates
            hs = (C.c_void_p * 1)(m.h.value)
            assert lib.l2b_verify_sample_ragged(hs, 1, (C.c_int32 * 1)(2), (C.c_int32 * 2)(1, 2), (C.c_int32 * 1)(3),
                                                (C.c_float * 1)(1.0), (C.c_float * 1)(0.9), None, None, 0, None) == -1
            for t, (k, v) in zip(ss, before):
                kk, vv = caches(t)
                assert np.array_equal(k, kk) and np.array_equal(v, vv)
            for t in ss:
                appended_is(l2b, t, P, 1)
        finally:
            close_all(ss[1:])


# ---- stream exactness -----------------------------------------------------------------------------------

SETTINGS = [(0.7, 0.0, True), (1.0, 0.9, False), (0.7, 0.9, True), (1.0, 0.0, False)]
SPEC_CASES = [(n, k) for n in ("S", "B") for k in ("own", "other", "near")]


@pytest.mark.parametrize("name,kind", SPEC_CASES, ids=[f"{n}-{k}" for n, k in SPEC_CASES])
def test_speculative_sample_equals_the_plain_loop(l2b, host, name, kind):
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    p, n = 230, 40                                     # crosses the 256-position attention split
    toks = stream(0, S, V)
    with l2b_env({}), l2b.Transformer(ck) as m:
        twin = m.session()
        draft, owned = make_draft(l2b, kind, m, name)
        try:
            for si, (temp, top_p, bos) in enumerate(SETTINGS):
                seed = 17 + si
                twin.reset()
                twin.prefill(toks[:p], 0, want_logits=False)
                want = plain_stream(l2b, host, twin, toks[p], p, n, temp, top_p, bos, seed=seed)
                want_rows = rows(twin, p + len(want))
                for k in (0, 1, 3, 8):
                    where = (temp, top_p, bos, k)
                    for t in (m, draft):
                        t.reset()
                        t.prefill(toks[:p], 0, want_logits=False)
                    got, rounds = speculative(host, m, draft, toks[p], p, n, k, temp, top_p, bos, seed=seed)
                    assert got == want, where
                    assert_rows(rows(m, p + len(got)), want_rows, where)
                    assert -(-len(got) // (k + 1)) <= rounds <= len(got), (where, rounds)
                    if kind == "own" and name == "S":  # single steps everywhere: every proposal is accepted
                        assert rounds == -(-len(got) // (k + 1)), (where, rounds)
                        assert_rows(rows(draft, p + len(got)), want_rows, where)
                    for t in (m, draft):           # both hold the stream's rows: pos + n_done is reachable
                        t.forward(1, p + len(got))
        finally:
            close_all([twin] + owned)


@pytest.mark.parametrize("name", ["S", "B"])
def test_two_calls_and_the_end_of_the_context(l2b, host, name):
    ck = payload(l2b, name)
    V, S = ck.vocab_size, ck.seq_len
    p = 20
    toks = stream(1, S, V)
    with l2b_env({}), l2b.Transformer(ck) as m:
        twin = m.session()
        near, owned = make_draft(l2b, "near", m, name)
        try:
            twin.prefill(toks[:p], 0, want_logits=False)
            want = plain_stream(l2b, host, twin, toks[p], p, 60, 1.0, 0.9, False, seed=5)
            # the PRNG continues where the plain loop leaves it: one more plain token after the stream
            extra = plain_stream(l2b, host, twin, want[-1], p + 60, 1, 1.0, 0.9, False)
            for t in (m, near):
                t.reset()
                t.prefill(toks[:p], 0, want_logits=False)
            a, _ = speculative(host, m, near, toks[p], p, 25, 3, 1.0, 0.9, False, seed=5)
            b, _ = speculative(host, m, near, a[-1], p + 25, 35, 3, 1.0, 0.9, False)
            assert a + b == want
            assert_rows(rows(m, p + 60), rows(twin, p + 60), "two calls")
            assert plain_stream(l2b, host, m, b[-1], p + 60, 1, 1.0, 0.9, False) == extra
            # the end of the context: at most seq_len - pos tokens
            for t in (twin, m, near):
                t.reset()
                t.prefill(toks[:S - 6], 0, want_logits=False)
            want = plain_stream(l2b, host, twin, toks[S - 6], S - 6, 50, 1.0, 0.9, False, seed=6)
            got, _ = speculative(host, m, near, toks[S - 6], S - 6, 50, 8, 1.0, 0.9, False, seed=6)
            assert got == want and len(got) == 6
        finally:
            close_all([twin] + owned)


def test_speculative_sample_refusals(l2b, host):
    ck = payload(l2b, "S")
    with l2b_env({}), l2b.Transformer(ck) as m:
        d = m.session()
        try:
            out, done = (C.c_int32 * 4)(), C.c_int32()
            f = host.l2h_generate_speculative_sample
            cfg = C.byref(m.cfg)
            assert f(m.h, cfg, m.h, cfg, 1, 0, 4, 3, 1.0, 0.9, 1, out, C.byref(done), None) == -1   # draft is target
            assert f(m.h, cfg, d.h, cfg, 1, 0, 4, 3, 0.0, 0.9, 1, out, C.byref(done), None) == -1   # temperature 0
            assert f(m.h, cfg, d.h, cfg, 1, 0, 4, 33, 1.0, 0.9, 1, out, C.byref(done), None) == -1  # k too large
            assert f(m.h, cfg, d.h, cfg, 1, 0, 4, 3, 1.0, 0.9, 1, None, C.byref(done), None) == -1
        finally:
            d.close()


def test_stories15m_target(l2b, host, stories15m):
    """The stories15M checkpoint as target from BOS: its own model (k = 3) and a stories15M-shaped model of
    another seed (k = 1, 3) as drafts."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    with l2b.Transformer(ck) as m, \
            l2b.Transformer(shape_checkpoint((288, 768, 6, 6, 6, 32000, 256)), synthetic_seed=11) as other:
        twin, own = m.session(), m.session()
        try:
            want = plain_stream(l2b, host, twin, 1, 0, 256, 1.0, 0.9, True, seed=42)
            for draft, k in ((own, 3), (other, 1), (other, 3)):
                m.reset()
                draft.reset()
                got, rounds = speculative(host, m, draft, 1, 0, 256, k, 1.0, 0.9, True, seed=42)
                assert got == want, k
                assert rounds <= len(got)
                if draft is own:
                    assert rounds == -(-len(got) // (k + 1))
        finally:
            close_all([twin, own])


def test_demo_draft_prints_the_device_sampler_text(stories15m, tokenizer_path):  # noqa: F811
    exe = os.path.join(ROOT, "llama2.zig_b200", "bin", "llama2_b200")
    base = [exe, stories15m, "-t", "1.0", "-p", "0.9", "-s", "42", "-z", tokenizer_path]
    plain = subprocess.run(base + ["--device-sampler"], capture_output=True, check=True, timeout=300).stdout
    for k in ("3", "0"):
        drafted = subprocess.run(base + ["--draft", stories15m, "--draft-k", k], capture_output=True, check=True,
                                 timeout=300).stdout
        assert drafted == plain, k
    assert len(plain) > 0
