"""GPU: the paged KV layout.  A paged context returns exactly what a contiguous context of the same payload,
weight format and KV format returns (its twin), after any sequence of forks, rewinds, resets, copies-on-write
and page recycling.  Only the row addresses differ: every paged kernel is the contiguous kernel the shape
selects.  Rows at and past a session's appended count are not defined in a paged context, so the caches are
compared below that count.

  1  twin: every test_gpu_variants case on the single-context paths; S and B with bf16 and q8 weights and
     with bf16 and round-bf16 KV.
  2  page boundaries: runs that end at and cross P-1, P, P+1 and 2P; prefill and ragged chunks that straddle
     a page boundary; a batched pass of 4 sessions at different page offsets (S: seq_len 300, B: 600).
  3  the batched calls on paged sessions, generate_argmax_batch with a stop, and generate_speculative with
     the target paged, the draft paged, and both.
  4  fork sharing: n_pos in {0, 1, P-1, P, P+1, 3P+5, seq_len} to 1, 3 and 9 destinations, a fork of a fork,
     and a fork onto sessions that held pages; every destination then continues with its own tokens and
     equals its twin; src is unchanged; pages_in_use follows a host model of the policy (PoolModel).
  5  copy-on-write: after a fork one destination rewinds into a shared page through forward, prefill,
     score, a rejecting verify and generate_argmax; src and the siblings stay bit-identical.
  6  recycled pages: sessions fill pages with another stream and are reset or destroyed; clean sessions
     that reuse those pages (they are not cleared) run the single, batched, verify and fork paths and equal
     clean contiguous twins.
  7  pool limit: with a cap, a call that needs a page returns OOM and changes no session; after another
     session is reset the same call succeeds; a cap below the pages in use is refused.
  8  accounting: page_bytes, kv_info bytes, sessions of a paged model are paged, and an emptied model holds
     no page.
  9  slow, llama2-7B: best-of-8 from a 1984-token prompt at seq_len 2048 in bf16 KV: tokens equal the
     contiguous twin's and the pool holds 47 pages.
 10  long context: L7, L3 and F128 of test_gpu_long_context (default; L2B_FUSE=0 L2B_ATTN=3pass on L7 and
     L3) in f32, bf16 and e4m3 (stress scales) KV, through test_gpu_long_context.check_twin: forward at
     the checked positions, the prefill chunks around last_short, score, forward_batch / forward_ragged /
     verify_argmax_ragged at per-query T, forks at 3, 299, last_short and 4000 rows.  Flash splits of up to
     911 rows over 16 staged pages, attn_wo_kernel's 8 cluster splits of 512 rows, the 3-pass kernel's
     456 / 911-row score buffers.  The envelope shapes and the paged seq_len limits are in
     test_gpu_envelope.
"""
import numpy as np
import pytest

import test_gpu_long_context as LC
from test_gpu_bf16 import _eq
from test_gpu_transformer import teacher_tokens
from test_gpu_variants import CASES, MODELS, l2b_env, payload

pytestmark = pytest.mark.gpu

P = 64


def twin(l2b, ck, env=None, weight_format="f32", kv_format="f32", seed=None):
    """(paged context, its contiguous twin) of ck under env (seed: device-synthesized weights)."""
    with l2b_env(env or {}):
        a = l2b.Transformer(ck, seed, weight_format=weight_format, kv_format=kv_format, kv_layout="paged")
        b = l2b.Transformer(ck, seed, weight_format=weight_format, kv_format=kv_format)
    return a, b


def rows(t, name, n, ck):
    """cache `name` of t, rows [0, n) of every layer"""
    c = t.state(name).reshape(ck.n_layers, ck.seq_len, -1)
    return c[:, :n]


def same_rows(a, b, n, what=""):
    for s in ("key_cache", "value_cache"):
        _eq(rows(a, s, n, a.ck), rows(b, s, n, b.ck), f"{what} {s} below {n}")


def pages_held(t):
    return t.kv_info()[1] // t.kv_pool_info()["page_bytes"]


def check_single(a, b, n, check, n_prompt):
    toks = teacher_tokens(n, a.ck.vocab_size)
    for pos, tok in enumerate(toks):
        la, lb = a.forward(tok, pos), b.forward(tok, pos)
        if pos in check:
            _eq(la, lb, f"logits at {pos}")
    same_rows(a, b, n, "forward")
    for s in ("x", "logits"):
        _eq(a.state(s), b.state(s), s)
    assert pages_held(a) == -(-n // P)
    for pos in check[:3]:
        assert a.forward_argmax(toks[pos], pos) == b.forward_argmax(toks[pos], pos)
    a.reset(); b.reset()
    assert a.kv_pool_info()["pages_in_use"] == 0
    forced = np.concatenate([np.array(toks[1:9], np.int32), np.full(8, -1, np.int32)])
    _eq(a.generate_argmax(toks[0], 0, 16, forced=forced, stop_on_bos=False),
        b.generate_argmax(toks[0], 0, 16, forced=forced, stop_on_bos=False), "generate_argmax")
    a.reset(); b.reset()
    _eq(a.prefill(toks[:n_prompt]), b.prefill(toks[:n_prompt]), "prefill logits")
    same_rows(a, b, n_prompt, "prefill")
    pa, ca = a.forward_sample(toks[n_prompt], n_prompt, 0.8, 0.9)
    pb, cb = b.forward_sample(toks[n_prompt], n_prompt, 0.8, 0.9)
    _eq(pa, pb, "forward_sample probs")
    assert (ca is None) == (cb is None) and (ca is None or np.array_equal(ca, cb))
    a.reset(); b.reset()
    la, ga = a.score(toks[:n_prompt])
    lb, gb = b.score(toks[:n_prompt])
    _eq(la, lb, "score log-probs")
    _eq(ga, gb, "score greedy")


@pytest.mark.parametrize("name,case,env", [(m, c, e) for m, c, e, _ in CASES],
                         ids=[f"{m}-{c}" for m, c, _, _ in CASES])
def test_twin(l2b, name, case, env):
    _, _, n, check, n_prompt = MODELS[name]
    a, b = twin(l2b, payload(l2b, name), env)
    with a, b:
        check_single(a, b, n, check, n_prompt)


@pytest.mark.parametrize("wf,kv", [("bf16", "f32"), ("q8", "f32"), ("f32", "bf16"), ("bf16", "bf16"),
                                   ("f32", "f32-round-bf16")])
@pytest.mark.parametrize("name", ["S", "B"])
def test_twin_formats(l2b, name, wf, kv):
    _, _, n, check, n_prompt = MODELS[name]
    a, b = twin(l2b, payload(l2b, name), weight_format=wf, kv_format=kv)
    with a, b:
        assert a.kv_info()[0] == kv and a.weight_info()[0] == wf
        check_single(a, b, n, check, n_prompt)


@pytest.mark.parametrize("name", ["S", "B"])
def test_page_boundaries(l2b, name):
    ck = payload(l2b, name)
    a, b = twin(l2b, ck)
    with a, b:
        toks = teacher_tokens(2 * P + 3, ck.vocab_size)
        for end in (P - 1, P, P + 1, 2 * P, 2 * P + 2):          # runs that end at / cross the boundaries
            a.reset(); b.reset()
            _eq(a.prefill(toks[:end]), b.prefill(toks[:end]), f"prefill to {end}")
            _eq(a.forward(toks[end], end), b.forward(toks[end], end), f"step at {end}")
            same_rows(a, b, end + 1, f"end {end}")
            assert pages_held(a) == -(-(end + 1) // P)
        a.reset(); b.reset()
        for lo, hi in ((0, P - 3), (P - 3, P + 4), (P + 4, 2 * P + 1)):   # chunks straddling a boundary
            _eq(a.prefill(toks[lo:hi], lo), b.prefill(toks[lo:hi], lo), f"chunk {lo}..{hi}")
        same_rows(a, b, 2 * P + 1, "chunks")
        sa = [a.session() for _ in range(4)]
        sb = [b.session() for _ in range(4)]
        try:
            starts = [P - 2, P, 2 * P - 1, 5]                       # 4 sessions at different page offsets
            for i, p in enumerate(starts):
                sa[i].prefill(toks[:p], want_logits=False)
                sb[i].prefill(toks[:p], want_logits=False)
            t4 = toks[10:14]
            _eq(l2b.forward_batch(sa, t4, starts), l2b.forward_batch(sb, t4, starts), "batch at offsets")
            pos = [p + 1 for p in starts]
            runs = [toks[20:23], toks[23:27], toks[27:29], toks[29:30]]
            _eq(l2b.forward_ragged(sa, runs, pos), l2b.forward_ragged(sb, runs, pos), "ragged across pages")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            for x, y, n in zip(sa, sb, pos):
                same_rows(x, y, n, "batched sessions")
        finally:
            for s in sa + sb:
                s.close()


@pytest.mark.parametrize("wf,kv", [("f32", "f32"), ("bf16", "bf16")])
@pytest.mark.parametrize("name", ["S", "B"])
def test_batched(l2b, name, wf, kv):
    a, b = twin(l2b, payload(l2b, name), weight_format=wf, kv_format=kv)
    with a, b:
        toks = teacher_tokens(40, a.ck.vocab_size)
        sa = [a.session() for _ in range(4)]
        sb = [b.session() for _ in range(4)]
        try:
            assert all(s.kv_pool_info()["page_rows"] == P for s in sa)
            for i in range(4):
                sa[i].prefill(toks[:3 + i], want_logits=False)
                sb[i].prefill(toks[:3 + i], want_logits=False)
            pos = [3, 4, 5, 6]
            t4 = toks[10:14]
            _eq(l2b.forward_batch(sa, t4, pos), l2b.forward_batch(sb, t4, pos), "forward_batch")
            pos = [p + 1 for p in pos]
            _eq(l2b.forward_argmax_batch(sa, t4, pos), l2b.forward_argmax_batch(sb, t4, pos), "argmax_batch")
            pos = [p + 1 for p in pos]
            ra = l2b.forward_sample_batch(sa, t4, pos, [1.0, 0.7, 1.0, 0.5], [0.9, 1.0, 0.95, 0.5])
            rb = l2b.forward_sample_batch(sb, t4, pos, [1.0, 0.7, 1.0, 0.5], [0.9, 1.0, 0.95, 0.5])
            _eq(ra[0], rb[0], "sample_batch probs")
            pos = [p + 1 for p in pos]
            runs = [toks[0:1], toks[1:6], toks[6:9], toks[9:11]]
            _eq(l2b.forward_ragged(sa, runs, pos), l2b.forward_ragged(sb, runs, pos), "forward_ragged")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            _eq(l2b.forward_argmax_ragged(sa, runs, pos), l2b.forward_argmax_ragged(sb, runs, pos), "argmax_ragged")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            ra = l2b.forward_sample_ragged(sa, runs, pos, [1.0] * 4, [0.9] * 4)
            rb = l2b.forward_sample_ragged(sb, runs, pos, [1.0] * 4, [0.9] * 4)
            _eq(ra[0], rb[0], "sample_ragged probs")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            ga = l2b.generate_argmax_batch(sa, t4, pos, 6, stop_on_bos=False)
            gb = l2b.generate_argmax_batch(sb, t4, pos, 6, stop_on_bos=False)
            for x, y in zip(ga, gb):
                _eq(x, y, "generate_argmax_batch")
            pos = [p + 6 for p in pos]
            vruns = [[int(g[-1])] + list(toks[20:23]) for g in ga]
            va = l2b.verify_argmax_ragged(sa, vruns, pos)
            vb = l2b.verify_argmax_ragged(sb, vruns, pos)
            _eq(va[1], vb[1], "n_accept")
            for x, y in zip(va[0], vb[0]):
                _eq(x, y, "verify greedy")
            pos = [p + int(k) + 1 for p, k in zip(pos, va[1])]
            sa_ = l2b.verify_sample_ragged(sa, vruns, pos, [1.0] * 4, [0.9] * 4)
            sb_ = l2b.verify_sample_ragged(sb, vruns, pos, [1.0] * 4, [0.9] * 4)
            _eq(sa_[0], sb_[0], "verify_sample probs")
            _eq(sa_[2], sb_[2], "verify_sample n_cand")
            pos = [p + len(r) for p, r in zip(pos, vruns)]
            for x, y, n in zip(sa, sb, pos):
                same_rows(x, y, n, "batched")
                assert pages_held(x) == -(-n // P)
        finally:
            for s in sa + sb:
                s.close()


def test_generate_batch_stop_releases(l2b):
    """A session that stops on BOS early releases the pages its reservation took past its end."""
    ck = payload(l2b, "S")
    a, b = twin(l2b, ck)
    with a, b:
        toks = teacher_tokens(P, ck.vocab_size)
        sa = [a.session() for _ in range(2)]
        sb = [b.session() for _ in range(2)]
        try:
            for x, y in zip(sa, sb):
                x.prefill(toks[:P - 4], want_logits=False)
                y.prefill(toks[:P - 4], want_logits=False)
            forced = np.full((2, 3 * P), -1, np.int32)
            forced[0, 5] = 1                                   # session 0 emits BOS after its 6th step
            ga = l2b.generate_argmax_batch(sa, toks[:2], [P - 4] * 2, 3 * P, forced=forced, stop_on_bos=True)
            gb = l2b.generate_argmax_batch(sb, toks[:2], [P - 4] * 2, 3 * P, forced=forced, stop_on_bos=True)
            for x, y in zip(ga, gb):
                _eq(x, y, "generate_argmax_batch with a stop")
            ends = [P - 4 + len(g) for g in ga]
            assert ends[0] == P - 4 + 6
            for x, y, n in zip(sa, sb, ends):
                same_rows(x, y, n, "stopped")
                assert pages_held(x) == -(-n // P)
        finally:
            for s in sa + sb:
                s.close()


@pytest.mark.parametrize("paged", ["target", "draft", "both"])
def test_speculative(l2b, paged):
    ck = payload(l2b, "S")
    with l2b.Transformer(ck, kv_layout="paged" if paged != "draft" else "contiguous") as t, \
            l2b.Transformer(ck, kv_layout="paged" if paged != "target" else "contiguous") as d, \
            l2b.Transformer(ck) as t2, l2b.Transformer(ck) as d2:
        toks = teacher_tokens(P + 7, ck.vocab_size)
        for m in (t, d, t2, d2):
            m.prefill(toks[:P + 6], want_logits=False)
        out, rounds = t.generate_speculative(d, toks[P + 6], P + 6, 2 * P + 9, 4, stop_on_bos=False)
        out2, rounds2 = t2.generate_speculative(d2, toks[P + 6], P + 6, 2 * P + 9, 4, stop_on_bos=False)
        _eq(out, out2, "speculative tokens")
        assert rounds == rounds2
        n = P + 6 + len(out)
        same_rows(t, t2, n, "target")
        same_rows(d, d2, n, "draft")


class PoolModel:
    """The pool policy, restated: page j of a session is a shared object; fork shares src's full pages and
    gives each destination a fresh page for a partial last one; a write into a page shared by several
    holders privatises it; a page is freed when no session holds it."""

    def __init__(self):
        self.held = {}            # session -> list of page ids (None: not held)
        self.next = 0

    def new(self):
        self.next += 1
        return self.next

    def set_len(self, s, n, seq_len):
        pages = self.held.setdefault(s, [None] * -(-seq_len // P))
        for j in range(len(pages)):
            if j * P >= n:
                pages[j] = None
            elif pages[j] is None:
                pages[j] = self.new()

    def write(self, s, lo, hi, n_after, seq_len):
        pages = self.held[s]
        for j in range(lo // P, (min(hi, seq_len) - 1) // P + 1):
            if pages[j] is None or self.refs(pages[j]) > 1:
                pages[j] = self.new()
        self.set_len(s, n_after, seq_len)

    def fork(self, src, dsts, n_pos):
        for d in dsts:
            pages = [None] * len(self.held[src])
            for j in range(n_pos // P):
                pages[j] = self.held[src][j]
            if n_pos % P:
                pages[n_pos // P] = self.new()
            self.held[d] = pages

    def refs(self, page):
        return sum(p == page for pages in self.held.values() for p in pages)

    def in_use(self):
        return len({p for pages in self.held.values() for p in pages if p is not None})


def _fork_case(l2b, ck, n_pos, n_dst):
    a, b = twin(l2b, ck)
    S = ck.seq_len
    toks = teacher_tokens(S, ck.vocab_size)
    model = PoolModel()
    with a, b:
        da = [a.session() for _ in range(n_dst)]
        db = [b.session() for _ in range(n_dst)]
        try:
            if n_pos:
                a.prefill(toks[:n_pos], want_logits=False)
                b.prefill(toks[:n_pos], want_logits=False)
            model.set_len("src", n_pos, S)
            for i, (x, y) in enumerate(zip(da, db)):          # destinations that held pages before the fork
                x.prefill(toks[:7 + i], want_logits=False)
                model.set_len(i, 7 + i, S)
            src_before = [a.state(s) for s in ("key_cache", "value_cache")]
            l2b.fork(a, da, n_pos)
            l2b.fork(b, db, n_pos)
            model.fork("src", list(range(n_dst)), n_pos)
            assert a.kv_pool_info()["pages_in_use"] == model.in_use()
            for x, y in zip(da, db):
                same_rows(x, y, n_pos, f"fork {n_pos}")
            if n_pos < S:
                for i, (x, y) in enumerate(zip(da, db)):       # each continues with its own tokens
                    n = min(S - n_pos, 3 + i)
                    own = [int(t) for t in teacher_tokens(n + i, ck.vocab_size)[i:]]
                    _eq(x.prefill(own, n_pos), y.prefill(own, n_pos), f"destination {i} continues")
                    model.write(i, n_pos, n_pos + n, n_pos + n, S)
                    same_rows(x, y, n_pos + n, f"destination {i}")
                assert a.kv_pool_info()["pages_in_use"] == model.in_use()
            for s, before in zip(("key_cache", "value_cache"), src_before):
                _eq(rows(a, s, n_pos, ck), before.reshape(ck.n_layers, S, -1)[:, :n_pos], "src unchanged")
            if n_pos >= 2 and n_dst > 1:                       # a fork of a fork
                e = a.session()
                try:
                    l2b.fork(da[0], [e], n_pos - 1)
                    model.held["e"] = None
                    model.fork(0, ["e"], n_pos - 1)
                    assert a.kv_pool_info()["pages_in_use"] == model.in_use()
                    f = b.session()
                    try:
                        l2b.fork(db[0], [f], n_pos - 1)
                        same_rows(e, f, n_pos - 1, "fork of a fork")
                    finally:
                        f.close()
                finally:
                    e.close()
                    del model.held["e"]
        finally:
            for s in da + db:
                s.close()
        for i in range(n_dst):
            model.held.pop(i, None)
        assert a.kv_pool_info()["pages_in_use"] == model.in_use()
        a.reset()
        assert a.kv_pool_info()["pages_in_use"] == 0


@pytest.mark.parametrize("n_dst", [1, 3, 9])
@pytest.mark.parametrize("n_pos", [0, 1, P - 1, P, P + 1, 3 * P + 5, "S"])
def test_fork(l2b, n_pos, n_dst):
    ck = payload(l2b, "S")
    _fork_case(l2b, ck, ck.seq_len if n_pos == "S" else n_pos, n_dst)


@pytest.mark.parametrize("path", ["forward", "prefill", "score", "verify", "generate"])
def test_copy_on_write(l2b, path):
    ck = payload(l2b, "S")
    a, b = twin(l2b, ck)
    n_pos, rewind = 2 * P + 10, P + 20                        # the rewind lands in shared page 1
    toks = teacher_tokens(n_pos + 8, ck.vocab_size)
    other = [int(t) for t in teacher_tokens(12, ck.vocab_size)[::-1]]
    with a, b:
        a.prefill(toks[:n_pos], want_logits=False)
        b.prefill(toks[:n_pos], want_logits=False)
        da = [a.session() for _ in range(3)]
        db = [b.session() for _ in range(3)]
        try:
            l2b.fork(a, da, n_pos)
            l2b.fork(b, db, n_pos)
            before = a.kv_pool_info()["pages_in_use"]
            x, y = da[0], db[0]
            if path == "verify":
                run = other[:4]                                     # drafts the greedy model rejects
                ra = l2b.verify_argmax_ragged([x], [run], [rewind])
                rb = l2b.verify_argmax_ragged([y], [run], [rewind])
                _eq(ra[1], rb[1], "n_accept")
                end = rewind + int(ra[1][0]) + 1                    # the appended count shrinks: page 2 goes
                grown = 0
            else:
                calls = {"forward": lambda s: s.forward(other[0], rewind),
                         "prefill": lambda s: s.prefill(other[:5], rewind),
                         "score": lambda s: s.score(other[:6], rewind)[0],
                         "generate": lambda s: s.generate_argmax(other[0], rewind, 5, stop_on_bos=False)}
                _eq(calls[path](x), calls[path](y), f"{path} after the rewind")
                end, grown = n_pos, 1                               # a rewind keeps the appended count
            same_rows(x, y, end, f"{path} destination")
            # page 1 was privatised; with verify the private partial page 2 lies past the new end
            assert a.kv_pool_info()["pages_in_use"] == before + grown
            for x, y in ((a, b), (da[1], db[1]), (da[2], db[2])):   # src and siblings unchanged ...
                same_rows(x, y, n_pos, "untouched holder")
                _eq(x.forward(toks[n_pos], n_pos), y.forward(toks[n_pos], n_pos), "untouched holder continues")
        finally:
            for s in da + db:
                s.close()


def test_recycled_pages(l2b):
    """Pages other sessions filled are recycled uncleared; sessions that reuse them equal clean twins."""
    ck = payload(l2b, "S")
    S = ck.seq_len
    a, b = twin(l2b, ck)
    toks = teacher_tokens(S, ck.vocab_size)
    junk = [int(t) for t in teacher_tokens(S, ck.vocab_size)[::-1]]
    with a, b:
        dirty = [a.session() for _ in range(3)]
        for d in dirty:
            d.prefill(junk[:S - 1], want_logits=False)
        allocated = a.kv_pool_info()["pages_allocated"]
        dirty[0].reset()
        dirty[1].close()
        sa = [a.session() for _ in range(3)]
        sb = [b.session() for _ in range(3)]
        try:
            for x, y in zip(sa, sb):
                _eq(x.prefill(toks[:P + 5]), y.prefill(toks[:P + 5]), "prefill on recycled pages")
            pos = [P + 5] * 3
            _eq(l2b.forward_ragged(sa, [toks[:3]] * 3, pos), l2b.forward_ragged(sb, [toks[:3]] * 3, pos), "ragged")
            pos = [p + 3 for p in pos]
            _eq(sa[0].generate_argmax(toks[5], pos[0], 70, stop_on_bos=False),
                sb[0].generate_argmax(toks[5], pos[0], 70, stop_on_bos=False), "generate")
            _eq(sa[1].score(toks[:80], pos[1])[0], sb[1].score(toks[:80], pos[1])[0], "score")
            va = l2b.verify_argmax_ragged([sa[2]], [toks[:4]], [pos[2]])
            vb = l2b.verify_argmax_ragged([sb[2]], [toks[:4]], [pos[2]])
            _eq(va[1], vb[1], "verify")
            l2b.fork(sa[0], [sa[2]], P + 2)
            l2b.fork(sb[0], [sb[2]], P + 2)
            _eq(sa[2].forward(toks[9], P + 2), sb[2].forward(toks[9], P + 2), "after a fork onto recycled pages")
            assert np.all(np.isfinite(sa[2].state("logits")))
            assert a.kv_pool_info()["pages_allocated"] == allocated   # every page came from the free list
        finally:
            for s in sa + sb:
                s.close()
            dirty[0].close()
            dirty[2].close()


def test_pool_limit(l2b):
    ck = payload(l2b, "S")
    a, b = twin(l2b, ck)
    toks = teacher_tokens(3 * P, ck.vocab_size)
    with a, b:
        other = a.session()
        try:
            other.prefill(toks[:P + 1], want_logits=False)        # 2 pages
            a.prefill(toks[:P], want_logits=False)                # 1 full page: the next row needs a new one
            b.prefill(toks[:P], want_logits=False)
            assert a.kv_pool_info()["pages_in_use"] == 3
            with pytest.raises(l2b.L2BError) as e:
                a.kv_pool_limit(2)
            assert e.value.status == -1
            a.kv_pool_limit(3)
            before = [rows(a, s, P, ck) for s in ("key_cache", "value_cache")]
            calls = {
                "forward": lambda: a.forward(toks[P], P),
                "prefill": lambda: a.prefill(toks[P:P + 3], P),
                "score": lambda: a.score(toks[P:P + 4], P),
                "generate": lambda: a.generate_argmax(toks[P], P, 3, stop_on_bos=False),
                "ragged": lambda: l2b.forward_ragged([a], [toks[P:P + 2]], [P]),
                "verify": lambda: l2b.verify_argmax_ragged([a], [list(toks[P:P + 3])], [P]),
                "fork": lambda: l2b.fork(a, [other], P - 1),      # a fresh page for the partial one
            }
            for name, call in calls.items():
                with pytest.raises(l2b.L2BError) as e:
                    call()
                assert e.value.status == -5, name                 # L2B_ERR_OOM
                info = a.kv_pool_info()
                assert info["pages_in_use"] == 3 and info["pages_allocated"] <= 3, name
                assert pages_held(a) == 1 and pages_held(other) == 2, name
                for s, r in zip(("key_cache", "value_cache"), before):
                    _eq(rows(a, s, P, ck), r, name)
            other.reset()
            _eq(a.prefill(toks[P:P + 3], P), b.prefill(toks[P:P + 3], P), "after the reset")
            same_rows(a, b, P + 3, "after the reset")
            assert a.kv_pool_info()["pages_allocated"] <= 3
            a.kv_pool_limit(0)
        finally:
            other.close()


def test_accounting(l2b):
    ck = payload(l2b, "S")
    for kv, el in (("f32", 4), ("bf16", 2)):
        with l2b.Transformer(ck, kv_format=kv, kv_layout="paged") as a, l2b.Transformer(ck, kv_format=kv) as c:
            info = a.kv_pool_info()
            kv_dim = ck.dim // ck.n_heads * ck.n_kv_heads
            assert info["page_rows"] == P and info["page_bytes"] == 2 * ck.n_layers * P * kv_dim * el
            assert c.kv_pool_info() == {"page_rows": 0, "page_bytes": 0, "pages_in_use": 0, "pages_allocated": 0}
            with pytest.raises(l2b.L2BError) as e:
                c.kv_pool_limit(4)
            assert e.value.status == -2
            assert a.kv_info() == (kv, 0)
            toks = teacher_tokens(P + 3, ck.vocab_size)
            a.prefill(toks, want_logits=False)
            s = a.session()
            assert s.kv_pool_info()["page_rows"] == P
            l2b.fork(a, [s], P + 3)
            assert a.kv_info() == (kv, 2 * info["page_bytes"]) and s.kv_info() == (kv, 2 * info["page_bytes"])
            assert a.kv_pool_info()["pages_in_use"] == 3
            s.close()
            a.reset()
            assert a.kv_pool_info()["pages_in_use"] == 0


@pytest.mark.parametrize("kv", ["f32", "bf16", "e4m3"])
@pytest.mark.parametrize("name,env_name", LC.TWIN_PARAMS)
def test_twin_long_context(l2b, name, env_name, kv):
    """The Llama head geometry at 4096 / 8192 positions (test_gpu_long_context.check_twin): splits of up to
    911 rows staged over 16 pages, attn_wo_kernel's 8 cluster splits of 512 rows, the 3-pass kernel's
    456 / 911-row score buffers.  e4m3 runs with stress scales."""
    ck = LC.payload(l2b, name)
    a, b = twin(l2b, ck, LC.ENVS[env_name], kv_format=kv)
    with a, b:
        if kv == "e4m3":
            from test_gpu_kv_e4m3 import stress_scales
            for t in (a, b):
                t.set_kv_scales(stress_scales(l2b, ck))
        LC.check_twin(l2b, a, b, name, env_name)


@pytest.mark.slow
def test_best_of_8_llama2_7b(l2b):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint("llama2-7B")
    ck.seq_len = 2048
    n_prompt, n_new = 1984, 64
    toks = teacher_tokens(n_prompt, ck.vocab_size)
    outs = {}
    for layout in ("paged", "contiguous"):
        with l2b.Transformer(ck, synthetic_seed=7, weight_format="bf16", kv_format="bf16", kv_layout=layout) as m:
            m.prefill(toks, want_logits=False)                   # 31 full pages
            dst = [m.session() for _ in range(8)]
            try:
                l2b.fork(m, dst, n_prompt - 1)                   # 30 shared, 63 rows copied per sample
                forced = np.full((8, n_new), -1, np.int32)
                for i in range(8):
                    forced[i, 0] = (i * 97 + 11) % ck.vocab_size  # a different first sample per stream
                outs[layout] = l2b.generate_argmax_batch(dst, [toks[n_prompt - 1]] * 8, [n_prompt - 1] * 8,
                                                         n_new, forced=forced, stop_on_bos=False)
                if layout == "paged":
                    assert m.kv_pool_info()["pages_in_use"] == 31 + 8 * 2
            finally:
                for d in dst:
                    d.close()
    for x, y in zip(outs["paged"], outs["contiguous"]):
        _eq(x, y, "best-of-8 tokens")
