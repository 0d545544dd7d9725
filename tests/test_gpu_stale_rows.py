"""GPU: no decode path reads or writes the KV rows past a stream's end.

A session routinely holds cache rows it does not own: l2b_reset only forgets the appended count, l2b_fork
may shrink a stream, a verify call leaves rejected drafts behind, and l2b_generate_argmax_batch must not
append rows for a session that stopped.  Every result has to be independent of the rows at or past its
position, and some calls promise never to write them.  attention_flash_kernel loads the first rows of
split 0 before it reads the position and masks them afterwards; attention_kernel and attn_wo_kernel stop
at t1 = min(T, ..); skip_b keeps a stopped session from appending.  A zero row read with weight zero, or
with full weight on peaked scores, passes the other tests, so the rows here hold NaN: any arithmetic use
of one, 0 x NaN included, turns the result into NaN, and any write over one is visible bit for bit.

Poisoning goes through the public API.  Embedding row P of an unshared-classifier payload is set to NaN
while the model is created (the payload is restored at once); a session poisoned by prefill([P] * seq_len)
with logits has every KV row of every layer, and the run state prefill writes, at NaN.  Its clean twin is a
fresh session of the same model.  P is a token the streams here never use (on the 97-entry vocabularies
the teacher stream uses every token, so P is replaced there).  The checks:

  A  reads: the same call sequence on poisoned sessions and on their clean twins gives the same output
     bits, all finite, and the same KV rows [0, appended), bit for bit.  Paths: forward, forward_argmax,
     forward_sample (T 1.0 / 0.7, top-p 0 / 0.9), generate_argmax forced then free, prefill from 0 and
     continuing, score, the three batch calls on 4 sessions at 4 positions, the three ragged calls with a
     prompt cut next to decode steps, both verify calls with a draft P rejected at several indices (the
     rejected rows are then NaN, and the next call must ignore them), generate_argmax_batch with staggered
     starts and a forced BOS, generate_speculative and the host's sampled speculative loop with target and
     draft poisoned, fork from a poisoned source into poisoned destinations and a continuation.  Calls end
     at T in {1, 2, 3, NG - 1, NG, NG + 1, 2NG - 1, 2NG, 2NG + 1, 255, 256, 257, seq_len}, where NG =
     256 / LPR row groups of attention_flash_kernel (split 0 preloads rows up to 2NG - 1).  On S and B the
     poisoned session's teacher-forced logits and KV rows are also held to test_gpu_ref64's float64 bound.
  B  writes: after every call, the rows past what the call may write (header text) are still NaN.
  C  neighbours: token P in one session of a shared pass (its decode token, or the first, a middle or the
     last position of its run; slot 0-3) leaves every other session's outputs and KV rows as they are with
     a clean token there, and a call of fewer than 4 vectors straight after equals its clean twin.
  D  ops: NaN in the other heads' columns of keys / values and in the row padding of
     vector_weighted_sum_rows gives the zero-padded result bit for bit.

Cases: S (fused attn_wo_kernel, L2B_FUSE=0, 3-pass, 32 splits, no graphs), B (batched GEMM and batched
flash, position loop, 3-pass, 32 splits), hs28 (3-pass only), hs4 and hs256 (the two ends of the flash LPR
range) fused and not, and the envelope's mqa64 and ctx4096-h32.

What fails when the rule is broken (each change built alone, the file run once): an invalid row weighted
by zero in attention_flash_kernel's `update` instead of skipped fails every path on every case that runs the
flash kernel (S nofuse / 32 splits, B default / position loop / 32 splits, hs4, hs256 and ctx4096-h32 without
fusion); one row more in the last split of attention_kernel and attn_wo_kernel fails every case, and the
neighbour checks; a fork that copies row n_pos as well fails the fork path everywhere.
The whole file takes 128 s on one H100 80GB HBM3 (700 W), about 20 s of it the float64 run of B.
"""
import copy

import numpy as np
import pytest

from test_gpu_envelope import ENVELOPE
from test_gpu_fork import rows
from test_gpu_ops import ATTN_SHAPES, MORE_ATTN_SHAPES
from test_gpu_ref64 import ATTN_TOL, bound, err, kernel_class, kv_rows, reference
from test_gpu_sessions import caches, close_all
from test_gpu_speculative import rms_final_offset
from test_gpu_transformer import teacher_tokens
from test_gpu_variants import MODELS, l2b_env, payload
from test_gpu_verify_sample import host, speculative  # noqa: F401  (fixture)
import ref64

pytestmark = pytest.mark.gpu

FUSE0 = {"L2B_FUSE": "0"}
CASES = [("S", "default", {}), ("S", "nofuse", FUSE0), ("S", "attn-3pass", {"L2B_FUSE": "0", "L2B_ATTN": "3pass"}),
         ("S", "attn-min-chunk8", {"L2B_FUSE": "0", "L2B_ATTN_MIN_CHUNK": "8"}), ("S", "no-graph", {"L2B_NO_GRAPH": "1"}),
         ("B", "default", {}), ("B", "prefill-batch0", {"L2B_PREFILL_BATCH": "0"}), ("B", "attn-3pass", {"L2B_ATTN": "3pass"}),
         ("B", "attn-min-chunk8", {"L2B_ATTN_MIN_CHUNK": "8"}),
         ("hs28", "default", {}), ("hs4", "default", {}), ("hs4", "nofuse", FUSE0),
         ("hs256", "default", {}), ("hs256", "nofuse", FUSE0),
         ("mqa64", "default", {}), ("ctx4096-h32", "default", {}), ("ctx4096-h32", "nofuse", FUSE0)]
PATHS = ["forward", "generate", "prefill", "score", "batch", "ragged", "verify", "generate-batch", "speculative",
         "fork"]
SAMPLE = [(1.0, 0.0), (1.0, 0.9), (0.7, 0.0), (0.7, 0.9)]        # (temperature, top_p)


# ---- poisoned models and sessions ---------------------------------------------------------------------

_envelope = {}


def checkpoint(l2b, oracle, name):
    if name in MODELS:
        return payload(l2b, name)
    if name not in _envelope:
        from llama2_zig_b200.checkpoint import shape_checkpoint
        _envelope.clear()
        shape, seed = ENVELOPE[name][:2]
        ck = shape_checkpoint(shape)
        ck.data = oracle.synth_checkpoint(oracle.make_config(*ck.shape_tuple), ck.shared_weights, seed)
        _envelope[name] = ck
    return _envelope[name]


def poison_token(ck):
    """The largest token the teacher stream of the whole context leaves out, else vocab - 1 (replaced in it)."""
    used = set(teacher_tokens(ck.seq_len + 1, ck.vocab_size))
    free = [t for t in range(ck.vocab_size - 1, 1, -1) if t not in used]
    return free[0] if free else ck.vocab_size - 1


def clean_stream(ck, P, rot=0):
    """seq_len + 1 teacher tokens with P replaced by P - 1, rotated by rot."""
    toks = [P - 1 if t == P else t for t in teacher_tokens(ck.seq_len + 1, ck.vocab_size)]
    return toks[rot:] + toks[:rot]


def poisoned_model(l2b, ck, P, data=None):
    """A model of ck (or of `data`, a payload of ck's shape) with embedding row P at NaN.  The payload is
    restored as soon as l2b_create returns: the payload cache is shared with other modules."""
    assert not ck.shared_weights                  # with a shared classifier every logit P would be NaN
    pck = copy.copy(ck)
    if data is not None:
        pck.data = data
    row = pck.data[P * ck.dim:(P + 1) * ck.dim]
    saved = row.copy()
    row[:] = np.nan
    try:
        return l2b.Transformer(pck)
    finally:
        row[:] = saved


def bits(o):
    """Every array of a (nested) call result as (dtype, shape, bytes); None kept."""
    if o is None:
        return [None]
    if isinstance(o, (list, tuple)):
        return [b for x in o for b in bits(x)]
    a = np.asarray(o)
    return [(a.dtype.str, a.shape, a.tobytes())]


def floats(o):
    if isinstance(o, (list, tuple)):
        return [a for x in o for a in floats(x)]
    a = np.asarray(o) if o is not None else None
    return [a] if a is not None and a.dtype.kind == "f" else []


def same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


class Pair:
    """A session whose KV rows and run state are all NaN, and its clean twin (a fresh session of the same
    model), driven through the same calls.  Rows [0, eq) of the two must be equal bit for bit; rows [nan,
    seq_len) of the poisoned one must still be NaN."""

    def __init__(self, m, P):
        S = m.ck.seq_len
        self.p, self.c = m.session(), m.session()
        assert np.isnan(self.p.prefill([P] * S, 0)).all()
        for cache in caches(self.p):
            assert np.isnan(cache).all()
        self.eq = self.nan = 0

    def wrote(self, hi, eq=None):
        """A call may have written rows up to hi; rows [0, eq) (default: every row below hi) are now defined."""
        self.nan = max(self.nan, hi)
        self.eq = max(self.eq, hi) if eq is None else eq
        assert self.eq <= self.nan <= self.p.ck.seq_len

    def check(self, where):
        S = self.p.ck.seq_len
        for a, b in zip(rows(self.p, S), rows(self.c, S)):
            assert same_bits(a[:, :self.eq], b[:, :self.eq]), ("rows below eq", self.eq, where)
            bad = np.nonzero(~np.isnan(a[:, self.nan:]).all(axis=(0, 2)))[0]
            assert bad.size == 0, ("written past the stream", self.nan + bad[:8], where)

    def close(self):
        close_all([self.p, self.c])


def both(pairs, fn, finite=True):
    """fn on the poisoned sessions and on their twins: the same bits; every float finite unless finite is
    False.  Returns the poisoned sessions' result."""
    got = fn([x.p for x in pairs])
    want = fn([x.c for x in pairs])
    assert bits(got) == bits(want)
    if finite:
        for a in floats(got):
            assert np.isfinite(a).all()
    return got


def check_all(pairs, where):
    for i, x in enumerate(pairs):
        x.check((where, i))


def lanes_per_row(hs):
    hs4 = hs // 4
    return 8 if hs4 % 8 == 0 else 4 if hs4 % 4 == 0 else 2 if hs4 % 2 == 0 else 1


def stream_ends(ck):
    """The T (= pos + 1) classes where rows past T are loaded at all, and where the split count changes."""
    ng = 256 // lanes_per_row(ck.dim // ck.n_heads)
    S = ck.seq_len
    return sorted({t for t in (1, 2, 3, ng - 1, ng, ng + 1, 2 * ng - 1, 2 * ng, 2 * ng + 1, 255, 256, 257, S)
                   if 1 <= t <= S})


_model = {}


@pytest.fixture(scope="module", autouse=True)
def close_models():
    yield
    for m, _, _ in _model.values():
        m.close()
    _model.clear()


def model(l2b, oracle, name, case, env):
    """The poisoned model of a case, one at a time (the parameters are grouped by case)."""
    key = (name, case)
    if key not in _model:
        for m, _, _ in _model.values():
            m.close()
        _model.clear()
        ck = checkpoint(l2b, oracle, name)
        P = poison_token(ck)
        with l2b_env(env):
            _model[key] = (poisoned_model(l2b, ck, P), ck, P)
    return _model[key]


# ---- A and B: each path on poisoned sessions and their twins --------------------------------------------

def path_forward(l2b, oracle, m, P, ts, name, env):
    """Teacher-forced forward over the whole context; at every T class forward_argmax and forward_sample as
    well.  On S and B the poisoned logits and KV rows against float64."""
    ck = m.ck
    S = ck.seq_len
    toks = clean_stream(ck, P)
    if name in ("S", "B"):
        rck, run, (orc_logits, orc_k, orc_v) = reference(l2b, oracle, name, "synthetic")
        _, _, n, check, _ = MODELS[name]
        assert toks[:n] == teacher_tokens(n, ck.vocab_size)
        e_orc = max(err(orc_logits[p], run.logits[p]) for p in check)
        kclass = kernel_class(name, env)
        case = f"{name}-stale"
    x = Pair(m, P)
    try:
        for pos in range(S):
            lg = both([x], lambda s: s[0].forward(toks[pos], pos))
            x.wrote(pos + 1)
            if name in ("S", "B"):
                if pos in check:
                    bound("forward", case, kclass, err(lg, run.logits[pos]), e_orc)
                if pos == n - 1:
                    for c, r, o in zip(caches(x.p), (run.key_cache, run.value_cache), (orc_k, orc_v)):
                        r = kv_rows(r.reshape(-1), rck, n)
                        bound("kv", case, kclass, err(kv_rows(c, rck, n), r), err(kv_rows(o, rck, n), r))
            if pos + 1 in ts:
                both([x], lambda s: s[0].forward_argmax(toks[pos], pos))
                for temp, top_p in SAMPLE:
                    both([x], lambda s: s[0].forward_sample(toks[pos], pos, temp, top_p, with_count=True))
                x.check(("forward", pos + 1))
    finally:
        x.close()


def path_generate(l2b, m, P, ts):
    """generate_argmax from 0, forced along the stream up to each T class and free for two steps past it;
    the next call starts at T."""
    toks = clean_stream(m.ck, P)
    S = m.ck.seq_len
    x = Pair(m, P)
    try:
        cur = 0
        for T in ts:
            n = min(T - cur + 2, S - cur)
            forced = np.array(toks[cur + 1:T] + [-1] * (n - (T - 1 - cur)), dtype=np.int32)[:n]
            out = both([x], lambda s: s[0].generate_argmax(toks[cur], cur, n, forced=forced, stop_on_bos=False))
            assert len(out) == n
            x.wrote(cur + n)
            x.check(("generate", T))
            cur = T
    finally:
        x.close()


def path_prefill(l2b, m, P, ts):
    """prefill from 0, then continuing at an offset, in chunks that end at each T class."""
    toks = clean_stream(m.ck, P)
    x = Pair(m, P)
    try:
        cur = 0
        for T in ts:
            both([x], lambda s: s[0].prefill(toks[cur:T], cur))
            x.wrote(T)
            x.check(("prefill", T))
            cur = T
    finally:
        x.close()


def path_score(l2b, m, P, ts):
    """score from 0, then continuing: each call runs positions up to T - 1 and appends T positions."""
    toks = clean_stream(m.ck, P)
    x = Pair(m, P)
    try:
        cur = 0
        for T in ts:
            lp, greedy = both([x], lambda s: s[0].score(toks[cur:T + 1], cur))
            assert lp.size == T - cur
            x.wrote(T)
            x.check(("score", T))
            cur = T
    finally:
        x.close()


def path_batch(l2b, m, P, ts):
    """forward_batch, forward_argmax_batch and forward_sample_batch of 4 sessions at 4 positions (T - 1 of
    the T classes); each session's next call is at a later position."""
    ck = m.ck
    toks = clean_stream(ck, P)
    pairs = [Pair(m, P) for _ in range(4)]
    done = [0] * 4
    try:
        for r in range(0, len(ts), 4):
            pos = [T - 1 for T in ts[r:r + 4]]
            xs = pairs[:len(pos)]
            for i, (x, p) in enumerate(zip(xs, pos)):
                if p > done[i]:
                    both([x], lambda s: s[0].prefill(toks[done[i]:p], done[i], want_logits=False))
            tk = [toks[p] for p in pos]
            both(xs, lambda s: l2b.forward_batch(s, tk, pos))
            both(xs, lambda s: l2b.forward_argmax_batch(s, tk, pos))
            temp = [SAMPLE[i][0] for i in range(len(pos))]
            top_p = [SAMPLE[i][1] for i in range(len(pos))]
            both(xs, lambda s: l2b.forward_sample_batch(s, tk, pos, temp, top_p))
            for i, (x, p) in enumerate(zip(xs, pos)):
                x.wrote(p + 1)
                done[i] = p + 1
            check_all(xs, ("batch", pos))
    finally:
        for x in pairs:
            x.close()


def path_ragged(l2b, m, P, ts):
    """Session 0 takes the prompt in chunks cut at the T classes while session 1 decodes one position per
    call at T - 1 (prefilled up to there); the three ragged calls in turn."""
    ck = m.ck
    toks = clean_stream(ck, P)
    other = clean_stream(ck, P, rot=7)
    pairs = [Pair(m, P) for _ in range(2)]
    try:
        cur = bcur = 0
        for r, T in enumerate(ts):
            b = T - 1
            if b > bcur:
                both([pairs[1]], lambda s: s[0].prefill(other[bcur:b], bcur, want_logits=False))
            runs = [toks[cur:T], [other[b]]]
            pos0 = [cur, b]
            kind = r % 3
            if kind == 0:
                both(pairs, lambda s: l2b.forward_ragged(s, runs, pos0))
            elif kind == 1:
                both(pairs, lambda s: l2b.forward_argmax_ragged(s, runs, pos0))
            else:
                both(pairs, lambda s: l2b.forward_sample_ragged(s, runs, pos0, [1.0, 0.7], [0.9, 0.0]))
            pairs[0].wrote(T)
            pairs[1].wrote(T)
            check_all(pairs, ("ragged", T))
            cur, bcur = T, T
    finally:
        for x in pairs:
            x.close()


VERIFY_M = 4                                       # drafts per run


def verify_starts(ts, S):
    return sorted({min(T - 1, S - 1 - VERIFY_M) for T in ts})


def greedy_drafts(l2b, m, toks, p0, n):
    """n greedy tokens from (toks[p0], p0) on a clean session of m."""
    g = m.session()
    try:
        if p0:
            g.prefill(toks[:p0], 0, want_logits=False)
        out = g.generate_argmax(toks[p0], p0, n, stop_on_bos=False)
        assert len(out) == n
        return [int(t) for t in out]
    finally:
        g.close()


def path_verify(l2b, m, P, ts):
    """verify_argmax_ragged and verify_sample_ragged of 4 sessions whose drafts are the greedy stream with
    draft c replaced by P: the argmax call accepts c drafts and leaves NaN rows from p0 + c + 1 on, which the
    next call, at the session's appended position, must ignore.  The sample call's outputs past the P
    position are NaN in both twins; the continuation starts right after the last draft before P."""
    ck = m.ck
    S = ck.seq_len
    toks = clean_stream(ck, P)
    starts = verify_starts(ts, S)
    rejects = [0, 1, 3, VERIFY_M]                 # VERIFY_M: every draft accepted
    for sample in (False, True):
        pairs = [Pair(m, P) for _ in range(4)]
        try:
            for r in range(0, len(starts), 4):
                p0 = starts[r:r + 4]
                xs = pairs[:len(p0)]
                runs, cs, tainted = [], [], False
                for i, (x, p) in enumerate(zip(xs, p0)):
                    if p:                              # from 0: the last continuation ran an emitted token
                        both([x], lambda s: s[0].prefill(toks[:p], 0, want_logits=False))
                    g = greedy_drafts(l2b, m, toks, p, VERIFY_M + 1)
                    c = rejects[(r // 4 + i) % 4]
                    d = g[:VERIFY_M]
                    if P in g[:c + 1]:                 # the model itself emits P: reject with another token
                        tainted = True
                        if c < VERIFY_M:
                            d[c] = next(t for t in (g[c] + 1, g[c] + 2) if t % ck.vocab_size != P) % ck.vocab_size
                    elif c < VERIFY_M:
                        d[c] = P
                    runs.append([toks[p]] + d)
                    cs.append(c)
                if not sample:
                    greedy, acc = both(xs, lambda s: l2b.verify_argmax_ragged(s, runs, p0), finite=False)
                    assert acc.tolist() == cs, (p0, cs)
                    nxt = [int(gr[-1]) for gr in greedy]
                    for x, p, c in zip(xs, p0, cs):
                        x.wrote(p + VERIFY_M + 1, eq=p + c + 1)
                else:
                    temp = [SAMPLE[i][0] for i in range(len(p0))]
                    top_p = [SAMPLE[i][1] for i in range(len(p0))]
                    probs, cands, n_cand = both(xs, lambda s: l2b.verify_sample_ragged(s, runs, p0, temp, top_p),
                                                finite=False)
                    v = 0
                    for c in cs:                       # positions p0 .. p0 + c precede the P draft
                        assert tainted or np.isfinite(probs[v:v + c + 1]).all()
                        v += VERIFY_M + 1
                    nxt = [toks[p + c + 1] for p, c in zip(p0, cs)]
                    for x, p, c in zip(xs, p0, cs):
                        x.wrote(p + VERIFY_M + 1, eq=p + c + 1)
                check_all(xs, ("verify", sample, p0))
                # the next call continues at the accepted position, over the rejected (NaN) rows
                at = [p + c + 1 for p, c in zip(p0, cs)]
                live = [i for i, a in enumerate(at) if a < S]
                sub = [xs[i] for i in live]
                if not sub:
                    continue
                if sample:
                    both(sub, lambda s: l2b.forward_sample_batch(s, [nxt[i] for i in live], [at[i] for i in live],
                                                                 [1.0] * len(sub), [0.9] * len(sub)),
                         finite=not tainted)
                else:
                    both(sub, lambda s: l2b.forward_batch(s, [nxt[i] for i in live], [at[i] for i in live]),
                         finite=not tainted and P not in nxt)
                for i in live:
                    xs[i].wrote(at[i] + 1)
                check_all(sub, ("verify continuation", sample, p0))
        finally:
            for x in pairs:
                x.close()


def path_generate_batch(l2b, m, P, ts):
    """generate_argmax_batch of 4 sessions started at T - 1 of 4 T classes; session 1 is forced to BOS at
    its second step and stops there while the others go on."""
    ck = m.ck
    S = ck.seq_len
    toks = clean_stream(ck, P)
    n_steps = 10
    pairs = [Pair(m, P) for _ in range(4)]
    try:
        for r in range(0, len(ts), 4):
            pos = [T - 1 for T in ts[r:r + 4]]
            xs = pairs[:len(pos)]
            for x, p in zip(xs, pos):                 # from 0: earlier free-running rows may hold any token
                if p:
                    both([x], lambda s: s[0].prefill(toks[:p], 0, want_logits=False))
            forced = np.full((len(pos), n_steps), -1, np.int32)
            forced[0, :3] = [toks[min(pos[0] + j, S)] for j in (1, 2, 3)]
            if len(pos) > 1:
                forced[1, 1] = 1
            out = both(xs, lambda s: l2b.generate_argmax_batch(s, [toks[p] for p in pos], pos, n_steps, forced=forced,
                                                               stop_on_bos=True))
            for i, (x, p, o) in enumerate(zip(xs, pos, out)):
                assert 1 <= len(o) <= min(n_steps, S - p)
                assert ((o >= 0) & (o < ck.vocab_size)).all()
                x.wrote(p + len(o))
            if len(pos) > 1 and pos[1] + 2 <= S:
                assert len(out[1]) == 2 and out[1][1] == 1
            check_all(xs, ("generate-batch", pos))
    finally:
        for x in pairs:
            x.close()


def near_payload(ck, P):
    """The payload with a perturbed final rmsnorm (a draft that disagrees now and then) and row P at NaN."""
    data = ck.data.copy()
    off = rms_final_offset(ck)
    rng = np.random.default_rng(5)
    data[off:off + ck.dim] *= (1.0 + 0.2 * rng.standard_normal(ck.dim)).astype(np.float32)
    return data


def path_speculative(l2b, host, m, P, ts):
    """generate_speculative and the host's sampled speculative loop, target and draft poisoned: tokens equal
    the twins', rows past the furthest position a round may run stay NaN in both, and the target continues."""
    ck = m.ck
    S = ck.seq_len
    toks = clean_stream(ck, P)
    near = poisoned_model(l2b, ck, P, near_payload(ck, P))
    n, k = 9, 3
    try:
        for sampled in (False, True):
            for T in ts[:3] + ts[-4:]:
                p = T - 1
                if p >= S - 1:
                    continue
                t, d = Pair(m, P), Pair(near, P)
                try:
                    if p:
                        both([t], lambda s: s[0].prefill(toks[:p], 0, want_logits=False))
                        both([d], lambda s: s[0].prefill(toks[:p], 0, want_logits=False))
                    if sampled:
                        out = [speculative(host, tt, dd, toks[p], p, n, k, 1.0, 0.9, False, seed=3 + p)[0]
                               for tt, dd in ((t.p, d.p), (t.c, d.c))]
                        assert out[0] == out[1], p
                        got = out[0]
                    else:
                        a = t.p.generate_speculative(d.p, toks[p], p, n, k, stop_on_bos=False)
                        b = t.c.generate_speculative(d.c, toks[p], p, n, k, stop_on_bos=False)
                        assert bits(a) == bits(b), p
                        got = a[0].tolist()
                    assert len(got) == min(n, S - p)
                    hi = min(S, p + n)
                    t.wrote(hi, eq=p + len(got))
                    d.wrote(hi, eq=p + len(got))
                    t.check(("speculative", sampled, p))
                    d.check(("speculative draft", sampled, p))
                    q = p + len(got)
                    if q < S:
                        both([t], lambda s: s[0].forward(got[-1], q), finite=P not in got)
                finally:
                    t.close()
                    d.close()
    finally:
        near.close()


def path_fork(l2b, m, P, ts):
    """fork from a poisoned source holding a stream of seq_len - 1 positions into 3 poisoned destinations at
    each T class; the source does not change, the destinations' rows from n_pos on stay NaN, and a
    forward_batch continues them."""
    ck = m.ck
    S = ck.seq_len
    toks = clean_stream(ck, P)
    src = Pair(m, P)
    dst = [Pair(m, P) for _ in range(3)]
    try:
        both([src], lambda s: s[0].prefill(toks[:S - 1], 0, want_logits=False))
        src.wrote(S - 1)
        before = [caches(s) for s in (src.p, src.c)]
        for T in ts:                              # ascending: rows from T on are still NaN in every destination
            if T >= S:
                continue
            l2b.fork(src.p, [x.p for x in dst], T)
            l2b.fork(src.c, [x.c for x in dst], T)
            for s, b in zip((src.p, src.c), before):
                for got, want in zip(caches(s), b):
                    assert same_bits(got, want), ("source changed", T)
            for x in dst:
                x.wrote(T)
            check_all(dst, ("fork", T))
            both(dst, lambda s: l2b.forward_batch(s, [toks[T]] * 3, [T] * 3))
            for x in dst:
                x.wrote(T + 1)
            check_all(dst, ("fork continuation", T))
        src.check("fork source")
    finally:
        for x in [src] + dst:
            x.close()


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name,case,env", CASES, ids=[f"{n}-{c}" for n, c, _ in CASES])
def test_stale_rows(l2b, oracle, host, name, case, env, path):  # noqa: F811
    m, ck, P = model(l2b, oracle, name, case, env)
    ts = stream_ends(ck)
    with l2b_env(env):
        if path == "forward":
            path_forward(l2b, oracle, m, P, ts, name, env)
        elif path == "speculative":
            path_speculative(l2b, host, m, P, ts)
        else:
            {"generate": path_generate, "prefill": path_prefill, "score": path_score, "batch": path_batch,
             "ragged": path_ragged, "verify": path_verify, "generate-batch": path_generate_batch,
             "fork": path_fork}[path](l2b, m, P, ts)


# ---- C: a NaN vector in a shared pass reaches no other session ------------------------------------------

NEIGHBOUR_CASES = [("S", "default", {}), ("B", "default", {}), ("B", "prefill-batch0", {"L2B_PREFILL_BATCH": "0"})]
CALLS = ["forward_batch", "forward_argmax_batch", "forward_sample_batch", "forward_ragged", "forward_argmax_ragged",
         "forward_sample_ragged", "verify_argmax_ragged", "verify_sample_ragged", "generate_argmax_batch"]
WHERE = {"decode": None, "first": 0, "middle": 2, "last": 4}    # where P sits in a run of 5 (None: a decode step)
RUN_LENS = (3, 1, 6, 2)                                          # the other sessions' runs


def call(l2b, kind, sess, runs, pos0):
    """One shared pass of `kind`; returns per session the outputs to compare (bits) and its token ids."""
    n = len(sess)
    temp, top_p = [SAMPLE[i % 4][0] for i in range(n)], [SAMPLE[i % 4][1] for i in range(n)]
    lens = [len(r) for r in runs]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(int)
    if kind in ("forward_batch", "forward_argmax_batch", "forward_sample_batch", "generate_argmax_batch"):
        tk = [r[0] for r in runs]
        if kind == "forward_batch":
            out = l2b.forward_batch(sess, tk, pos0)
            return [[out[i]] for i in range(n)], [[]] * n
        if kind == "forward_argmax_batch":
            out = l2b.forward_argmax_batch(sess, tk, pos0)
            return [[out[i]] for i in range(n)], [[int(out[i])] for i in range(n)]
        if kind == "forward_sample_batch":
            probs, cands, nc = l2b.forward_sample_batch(sess, tk, pos0, temp, top_p)
            return [[probs[i], cands[i], nc[i]] for i in range(n)], [[]] * n
        out = l2b.generate_argmax_batch(sess, tk, pos0, 4, stop_on_bos=False)
        return [[o] for o in out], [o.tolist() for o in out]
    if kind == "forward_ragged":
        out = l2b.forward_ragged(sess, runs, pos0)
        return [[out[i]] for i in range(n)], [[]] * n
    if kind == "forward_argmax_ragged":
        out = l2b.forward_argmax_ragged(sess, runs, pos0)
        return [[out[i]] for i in range(n)], [[int(out[i])] for i in range(n)]
    if kind == "forward_sample_ragged":
        probs, cands, nc = l2b.forward_sample_ragged(sess, runs, pos0, temp, top_p)
        return [[probs[i], cands[i], nc[i]] for i in range(n)], [[]] * n
    if kind == "verify_argmax_ragged":
        greedy, acc = l2b.verify_argmax_ragged(sess, runs, pos0)
        return [[greedy[i], acc[i]] for i in range(n)], [greedy[i].tolist() for i in range(n)]
    probs, cands, nc = l2b.verify_sample_ragged(sess, runs, pos0, temp, top_p)
    return ([[probs[offs[i]:offs[i + 1]], cands[offs[i]:offs[i + 1]], nc[offs[i]:offs[i + 1]]] for i in range(n)],
            [[]] * n)


def appended_after(kind, runs, pos0, outs):
    """Positions each session holds after the call (verify_argmax: its accepted position)."""
    if kind == "verify_argmax_ragged":
        return [p + int(o[1]) + 1 for p, o in zip(pos0, outs)]
    if kind == "generate_argmax_batch":
        return [p + 4 for p in pos0]
    return [p + len(r) for p, r in zip(pos0, runs)]


@pytest.mark.parametrize("kind", CALLS)
@pytest.mark.parametrize("name,case,env", NEIGHBOUR_CASES, ids=[f"{n}-{c}" for n, c, _ in NEIGHBOUR_CASES])
def test_neighbours(l2b, oracle, name, case, env, kind):
    m, ck, P = model(l2b, oracle, name, case, env)
    S, V = ck.seq_len, ck.vocab_size
    toks = clean_stream(ck, P)
    Q = toks[3]
    p0 = 250                                      # the runs cross the 256-position attention split
    decode_only = kind in ("forward_batch", "forward_argmax_batch", "forward_sample_batch", "generate_argmax_batch")
    wheres = ["decode"] if decode_only else (["first", "middle", "last"] if kind.startswith("verify")
                                              else list(WHERE))
    with l2b_env(env):
        src = m.session()
        A = [m.session() for _ in range(4)]
        B = [m.session() for _ in range(4)]
        try:
            src.prefill(toks[:p0], 0, want_logits=False)
            for slot in range(4):
                for where in wheres:
                    l2b.fork(src, A + B, p0)
                    runs = [clean_stream(ck, P, rot=17 * (i + 1))[:RUN_LENS[i]] for i in range(4)]
                    runs[slot] = clean_stream(ck, P, rot=5)[:1 if WHERE[where] is None else 5]
                    if decode_only:
                        runs = [r[:1] for r in runs]
                    clean = [list(r) for r in runs]
                    runs[slot][WHERE[where] or 0] = P
                    pos0 = [p0] * 4
                    got, ids = call(l2b, kind, A, runs, pos0)
                    want, _ = call(l2b, kind, B, clean, pos0)
                    others = [i for i in range(4) if i != slot]
                    for i in others:
                        assert bits(got[i]) == bits(want[i]), (slot, where, i)
                    assert all(0 <= t < V for t in ids[slot]), (slot, where, ids[slot])
                    held = appended_after(kind, runs, pos0, got)
                    for i in others:
                        hi = min(held[i], S)
                        for a, b in zip(rows(A[i], hi), rows(B[i], hi)):
                            assert same_bits(a, b), (slot, where, i)
                    # fewer than 4 vectors straight after the pass that carried NaN
                    nxt = [i for i in others if held[i] < S][:3 if slot % 2 else 2]
                    tk = [toks[held[i]] for i in nxt]
                    at = [held[i] for i in nxt]
                    a = l2b.forward_batch([A[i] for i in nxt], tk, at)
                    b = l2b.forward_batch([B[i] for i in nxt], tk, at)
                    assert same_bits(a, b) and np.isfinite(a).all(), (slot, where)
                    a = l2b.forward_sample_ragged([A[i] for i in nxt], [[t] for t in tk], at, [0.7] * len(nxt),
                                                  [0.9] * len(nxt))
                    b = l2b.forward_sample_ragged([B[i] for i in nxt], [[t] for t in tk], at, [0.7] * len(nxt),
                                                  [0.9] * len(nxt))
                    assert bits(a) == bits(b), (slot, where)
        finally:
            close_all([src] + A + B)


# ---- D: other heads' columns and row padding at the op level ---------------------------------------------

@pytest.mark.parametrize("attn", ["default", "3pass"])
@pytest.mark.parametrize("hs,stride,npos", ATTN_SHAPES + MORE_ATTN_SHAPES)
def test_attention_head_ignores_other_columns(l2b, monkeypatch, hs, stride, npos, attn):
    """keys / values columns [hs, stride) are the other kv heads' in the real layout: NaN there gives the
    zero-padded result bit for bit, within ATTN_TOL of float64."""
    if attn == "3pass":
        monkeypatch.setenv("L2B_ATTN", "3pass")
    else:
        monkeypatch.delenv("L2B_ATTN", raising=False)
    rng = np.random.default_rng(hs * 13 + npos)
    q = rng.standard_normal(hs).astype(np.float32)
    keys = np.zeros((npos, stride), np.float32)
    vals = np.zeros((npos, stride), np.float32)
    keys[:, :hs] = rng.standard_normal((npos, hs))
    vals[:, :hs] = rng.standard_normal((npos, hs))
    want = l2b.attention_head(q, keys, vals)
    keys[:, hs:] = np.nan
    vals[:, hs:] = np.nan
    got = l2b.attention_head(q, keys, vals)
    assert same_bits(got, want)
    sc = (keys[:, :hs].astype(np.float64) @ q.astype(np.float64)) / np.sqrt(np.float64(np.float32(hs)))
    assert err(got, ref64.softmax(sc) @ vals[:, :hs].astype(np.float64)) <= ATTN_TOL


@pytest.mark.parametrize("width,stride,n", [(3, 5, 3), (7, 9, 5), (48, 96, 300), (128, 512, 65), (4, 12, 1000)])
def test_weighted_sum_rows_ignores_padding(l2b, width, stride, n):
    rng = np.random.default_rng(width * 7 + n)
    rows_ = np.zeros((n, stride), np.float32)
    rows_[:, :width] = rng.standard_normal((n, width))
    w = rng.standard_normal(n).astype(np.float32)
    want = l2b.vector_weighted_sum_rows(np.zeros(width, np.float32), rows_.reshape(-1), stride, w)
    rows_[:, width:] = np.nan
    got = l2b.vector_weighted_sum_rows(np.zeros(width, np.float32), rows_.reshape(-1), stride, w)
    assert same_bits(got, want)
    ref = w.astype(np.float64) @ rows_[:, :width].astype(np.float64)
    assert np.max(np.abs(got - ref)) <= 1e-5 * (np.max(np.abs(ref)) + 1)
