"""GPU: beam search (l2b_beam_search) and its candidate kernel (l2b_op_logprob_topk).

  1  logprob_topk against an exact numpy restatement: ls = -logprob(argmax) is exact (l_max - m = 0), so
     lp_i = f32(f32(l_i - m) - ls) are the device's bits; the full order for k = 1 .. 16 on n in {16, 1000,
     32000, 128256}, with repeated maxima, ties made by rounding, -inf entries and huge spreads.  Every
     returned value equals l2b.logprob of its index bit for bit.
  2  the search against `ref_search`, which restates the rule of the header on a contiguous twin of the same
     payload: for every live hypothesis at every step it forks the twin's prompt, runs forward_ragged of
     [token, y_1 .. y_t] and takes logprob_topk of the logits.  Tokens, lengths, log-probabilities and n_run
     are equal bit for bit, and each beam's KV rows below its appended count equal the twin's fork + ragged
     rows.  Models S (single steps) and B (shared weight passes) of test_gpu_variants; B in {1, 2, 3, 4, 5,
     8}; stop_on_bos 0 and 1; prompts ending at 63, 64 and 127 (siblings copy a shared page at its
     boundary), and a pos near seq_len (T < n_steps).  On S and B also bf16 and q8 weights and bf16 KV.
  3  BOS: S with its classifier row 1 scaled, so BOS enters the top 2B at some steps; the reference shows F
     filling, a BOS past pool position B being dropped and the early stop, and the device matches there.
  4  pages: src's rows, pages and logits are unchanged; afterwards the pool holds at most src's pages plus
     each result's pages of rows [pos, pos + len); after the beams reset it holds src's pages alone.  Under a
     pool limit too small for the search the call returns OOM, src is unchanged, every beam has 0 positions
     appended and no page is lost; with the limit raised the same call equals the reference.  The argument
     refusals, n_steps == 0 and a contiguous model.
  5  the demo's --beam prints the text of the best result of beam_search on the same checkpoint.
  6  slow, llama2-7B synthetic, bf16 weights, bf16 paged KV, 1984-token prompt, B = 4, 16 steps: equal to the
     reference; the pages held are printed.
"""
import os
import subprocess

import numpy as np
import pytest

from test_gpu_bf16 import _eq
from test_gpu_kv_bf16 import demo_text
from test_gpu_kv_paged import pages_held, rows
from test_gpu_transformer import teacher_tokens
from test_gpu_variants import MODELS, payload
from test_host_twin import tokenizer_path  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

P = 64
BOS = 1


# ---- 1: the candidate kernel -------------------------------------------------------------------------

def fkey(x):
    """argmax_key's order of a float32 (its high word): larger value, larger key."""
    u = int(np.float32(x).view(np.uint32))
    return (~u & 0xFFFFFFFF) if u & 0x80000000 else (u | 0x80000000)


def topk_restated(l2b, logits, k):
    """(lp, index) of the k best, best first: lp_i = f32(f32(l_i - m) - ls), ls = -logprob(argmax) (exact:
    l_max - m = 0), ordered by argmax_key(lp, i)."""
    x = np.asarray(logits, np.float32)
    m = np.float32(x.max())
    ls = -l2b.logprob(x, int(np.argmax(x)))
    lp = ((x - m).astype(np.float32) - ls).astype(np.float32)
    order = sorted(range(x.size), key=lambda i: (-fkey(lp[i]), i))[:k]
    return lp[order], np.array(order, np.int32)


def topk_rows(n, rng):
    rows_ = {"normal": (rng.standard_normal(n) * 3).astype(np.float32)}
    r = rng.standard_normal(n).astype(np.float32)
    top = rng.choice(n, size=min(n, 5), replace=False)
    r[top] = r.max() + 1                                         # repeated maxima
    rows_["repeated-max"] = r
    # near-equal logits whose differences vanish under - ls (ls = log(sum) ~ log(n)): the larger logit
    # sits at the larger index, so an order on the logits would differ from the order on lp
    r = np.full(n, 1.0, np.float32) - np.float32(2.0 ** -20) * rng.integers(20, 40, n).astype(np.float32)
    r[np.arange(min(n, 12))] = np.float32(1.0) - np.float32(2.0 ** -24) * np.arange(min(n, 12))[::-1]
    rows_["rounding-ties"] = r
    r = (rng.standard_normal(n) * 5).astype(np.float32)
    r[rng.choice(n, size=n // 3, replace=False)] = -np.inf     # -inf entries
    rows_["minus-inf"] = r
    r = (rng.standard_normal(n) * 1e30).astype(np.float32)      # huge spread: most exp() underflow
    rows_["huge-spread"] = r
    return rows_


@pytest.mark.parametrize("n", [16, 1000, 32000, 128256])
def test_logprob_topk(l2b, n):
    rng = np.random.default_rng(n)
    ties_seen = False
    for kind, x in topk_rows(n, rng).items():
        want_lp, want_ix = topk_restated(l2b, x, min(16, n))
        ties_seen |= bool(np.any(want_lp[1:] == want_lp[:-1]))
        for k in range(1, min(16, n) + 1):
            got = l2b.logprob_topk(x, k)
            _eq(got["index"], want_ix[:k], f"{kind} n={n} k={k} indices")
            _eq(got["prob"], want_lp[:k], f"{kind} n={n} k={k} lp")
        for lp, ix in zip(got["prob"], got["index"]):
            _eq(np.float32(lp), l2b.logprob(x, int(ix)), f"{kind} n={n}: logprob of {ix}")
    assert ties_seen, "no row had two candidates of one lp"


# ---- 2: the search against its restatement -------------------------------------------------------------

class Hyp:
    def __init__(self, toks, c, step, at):
        self.toks, self.c, self.step, self.at = toks, np.float32(c), step, at

    def norm(self):
        return np.float32(self.c / np.float32(len(self.toks)))

    def order(self):
        """the result order: larger normalised score, then larger c, then earlier creation"""
        return (-fkey(self.norm()), -fkey(self.c), self.step, self.at)


def ref_search(cands, token, n_beams, T, stop):
    """The rule of l2b_beam_search's header.  cands(runs) gives, for each live hypothesis's tokens [y_1 ..
    y_t], its K = 2B candidates (lp, index) best first.  Returns (tokens, logprobs, n_run, events)."""
    B, K = n_beams, 2 * n_beams
    live, fin = [Hyp([], 0.0, -1, 0)], []
    ev = {"finished": 0, "dropped": 0, "early": False}
    ran = 0
    for t in range(T):
        C = cands([h.toks for h in live])
        pool = [(np.float32(live[h].c + C[h][0][r]), h, r) for h in range(len(live)) for r in range(K)]
        pool.sort(key=lambda x: (-fkey(x[0]), x[1], x[2]))
        nxt = []
        for q, (score, h, r) in enumerate(pool):
            if len(nxt) == B:
                break
            y = Hyp(live[h].toks + [int(C[h][1][r])], score, t, q)
            if stop and y.toks[-1] == BOS:
                if q < B:
                    fin.append(y)
                    fin.sort(key=Hyp.order)
                    del fin[B:]
                    ev["finished"] += 1
                else:
                    ev["dropped"] += 1
                continue
            nxt.append(y)
        live = nxt
        ran = t + 1
        if stop and len(fin) == B and fin[-1].norm() >= np.float32(live[0].c / np.float32(t + 1)):
            ev["early"] = True
            break
    res = sorted(fin + live, key=Hyp.order)[:B]
    return [np.array(h.toks, np.int32) for h in res], np.array([h.c for h in res], np.float32), ran, ev


def twin_cands(l2b, twin, scratch, token, pos, K):
    """candidates of each run [token, y_1 .. y_t] at pos on a fork of the twin's prompt"""
    def cands(runs):
        d = scratch[:len(runs)]
        l2b.fork(twin, d, pos)
        logits = l2b.forward_ragged(d, [[token] + r for r in runs], [pos] * len(runs))
        out = []
        for row in logits:
            c = l2b.logprob_topk(row, K)
            out.append((c["prob"], c["index"]))
        return out
    return cands


class Pair:
    """a paged model (the device under test) and its contiguous twin, both with the same prompt"""

    def __init__(self, l2b, ck, n_prompt, n_beams, weight_format="f32", kv_format="f32"):
        self.l2b, self.ck, self.n_prompt = l2b, ck, n_prompt
        self.a = l2b.Transformer(ck, weight_format=weight_format, kv_format=kv_format, kv_layout="paged")
        self.b = l2b.Transformer(ck, weight_format=weight_format, kv_format=kv_format)
        self.toks = teacher_tokens(ck.seq_len, ck.vocab_size)
        self.a.prefill(self.toks[:n_prompt], want_logits=False)
        self.b.prefill(self.toks[:n_prompt], want_logits=False)
        self.beams = [self.a.session() for _ in range(n_beams)]
        self.scratch = [self.b.session() for _ in range(n_beams)]

    def close(self):
        for s in self.beams + self.scratch:
            s.close()
        self.a.close()
        self.b.close()

    def reference(self, pos, n_beams, n_steps, stop):
        T = min(n_steps, self.ck.seq_len - pos)
        cands = twin_cands(self.l2b, self.b, self.scratch, self.toks[pos], pos, 2 * n_beams)
        return ref_search(cands, self.toks[pos], n_beams, T, stop)

    def run(self, pos, n_beams, n_steps, stop):
        return self.l2b.beam_search(self.a, self.toks[pos], pos, self.beams[:n_beams], n_steps, stop_on_bos=stop)

    def check(self, pos, n_beams, n_steps, stop, what=""):
        """device == reference: tokens, lengths, log-probabilities, n_run, each beam's KV rows; src unchanged.
        Returns the reference's events."""
        before = [rows(self.a, s, self.n_prompt, self.ck) for s in ("key_cache", "value_cache")]
        held, logits = pages_held(self.a), self.a.state("logits")
        toks, lps, ran = self.run(pos, n_beams, n_steps, stop)
        want_toks, want_lps, want_ran, ev = self.reference(pos, n_beams, n_steps, stop)
        assert ran == want_ran, (what, ran, want_ran)
        assert len(toks) == n_beams
        for i in range(n_beams):
            _eq(toks[i], want_toks[i], f"{what} result {i} tokens")
        _eq(lps, want_lps, f"{what} logprobs")
        for s, r in zip(("key_cache", "value_cache"), before):
            _eq(rows(self.a, s, self.n_prompt, self.ck), r, f"{what} src {s}")
        assert pages_held(self.a) == held
        _eq(self.a.state("logits"), logits, f"{what} src logits")
        d = self.scratch[0]
        for i in range(n_beams):
            n = pos + len(toks[i])
            self.l2b.fork(self.b, [d], pos)
            if len(toks[i]):
                self.l2b.forward_ragged([d], [[self.toks[pos]] + [int(x) for x in toks[i][:-1]]], [pos])
            for s in ("key_cache", "value_cache"):
                _eq(rows(self.beams[i], s, n, self.ck), rows(d, s, n, self.ck), f"{what} beam {i} {s}")
        # the pool: src's pages and each result's pages of rows [pos, pos + len)
        bound = held + sum((pos + len(t) - 1) // P - pos // P + 1 for t in toks if len(t))
        assert self.a.kv_pool_info()["pages_in_use"] <= bound, what
        # each beam continues its hypothesis where it ends
        for i in range(n_beams):
            if len(toks[i]) and pos + len(toks[i]) < self.ck.seq_len:
                self.beams[i].forward(int(toks[i][-1]), pos + len(toks[i]))
                break
        return ev

    def reset_beams(self):
        for s in self.beams:
            s.reset()
        assert self.a.kv_pool_info()["pages_in_use"] == pages_held(self.a)


def make_pair(l2b, name, n_prompt, n_beams, **kw):
    return Pair(l2b, payload(l2b, name), n_prompt, n_beams, **kw)


@pytest.mark.parametrize("stop", [0, 1])
@pytest.mark.parametrize("n_beams", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("name", ["S", "B"])
def test_search(l2b, name, n_beams, stop):
    seq_len = MODELS[name][0][6]
    pr = make_pair(l2b, name, seq_len - 3, n_beams)
    try:
        for pos in (63, 64, 127, seq_len - 3):
            pr.check(pos, n_beams, 6, stop, f"{name} B={n_beams} stop={stop} pos={pos}")
            pr.reset_beams()
    finally:
        pr.close()


@pytest.mark.parametrize("wf,kv", [("bf16", "f32"), ("q8", "f32"), ("f32", "bf16")])
@pytest.mark.parametrize("name", ["S", "B"])
def test_search_formats(l2b, name, wf, kv):
    pr = make_pair(l2b, name, 130, 5, weight_format=wf, kv_format=kv)
    try:
        for pos, stop in ((127, 1), (64, 0)):
            pr.check(pos, 5, 6, stop, f"{name} {wf}/{kv} pos={pos}")
            pr.reset_beams()
    finally:
        pr.close()


# ---- 3: BOS ---------------------------------------------------------------------------------------------

BOS_SCALES = (4.0, 6.0)


def bos_checkpoint(l2b, scale):
    """S with classifier row 1 (BOS) scaled: BOS's logit swings far up or down with the sign of its dot."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    base = payload(l2b, "S")
    ck = shape_checkpoint(MODELS["S"][0])
    data = base.data.copy()
    wcls = data.size - ck.vocab_size * ck.dim
    data[wcls + ck.dim:wcls + 2 * ck.dim] *= np.float32(scale)
    ck.data = data
    return ck


def test_bos(l2b):
    seen = {"finished": 0, "dropped": 0, "early": 0}
    for scale in BOS_SCALES:
        ck = bos_checkpoint(l2b, scale)
        pr = Pair(l2b, ck, 200, 8)
        try:
            for n_beams in (1, 3, 8):
                for pos in (40, 127, 190):
                    ev = pr.check(pos, n_beams, 10, 1, f"bos x{scale} B={n_beams} pos={pos}")
                    pr.reset_beams()
                    seen["finished"] += ev["finished"]
                    seen["dropped"] += ev["dropped"]
                    seen["early"] += ev["early"]
        finally:
            pr.close()
    print("BOS events over the cases:", seen)
    assert seen["finished"] > 0 and seen["dropped"] > 0 and seen["early"] > 0, seen


# ---- 4: pages, the pool limit and refusals ---------------------------------------------------------------

def test_pool_limit(l2b):
    pr = make_pair(l2b, "S", 130, 4)
    try:
        a = pr.a
        pos = 100                                   # a partial page: the first step copies it
        src_pages = pages_held(a)
        assert a.kv_pool_info()["pages_in_use"] == src_pages
        before = [rows(a, s, 130, pr.ck) for s in ("key_cache", "value_cache")]
        a.kv_pool_limit(src_pages + 2)              # step 1 needs a page for each of the 4 children
        with pytest.raises(l2b.L2BError) as e:
            pr.run(pos, 4, 6, 0)
        assert e.value.status == -5                 # L2B_ERR_OOM
        info = a.kv_pool_info()
        assert info["pages_in_use"] == src_pages, info
        for s, r in zip(("key_cache", "value_cache"), before):
            _eq(rows(a, s, 130, pr.ck), r, f"src {s} after OOM")
        for bm in pr.beams:
            assert pages_held(bm) == 0
            with pytest.raises(l2b.L2BError) as e:   # 0 positions appended: position 1 skips ahead
                bm.forward(pr.toks[0], 1)
            assert e.value.status == -7
            bm.reset()
        a.kv_pool_limit(0)
        pr.check(pos, 4, 6, 0, "after the limit is raised")
        pr.reset_beams()
    finally:
        pr.close()


def test_refusals(l2b):
    pr = make_pair(l2b, "S", 70, 3)
    try:
        a, bm, t = pr.a, pr.beams, pr.toks
        V, S = pr.ck.vocab_size, pr.ck.seq_len
        other = l2b.Transformer(pr.ck, kv_layout="paged")
        bad = [
            (lambda: l2b.beam_search(a, t[5], 5, [], 4), -1),
            (lambda: l2b.beam_search(a, t[5], 5, bm + [a.session() for _ in range(6)], 4), -1),
            (lambda: l2b.beam_search(a, t[5], 5, [bm[0], bm[0]], 4), -1),
            (lambda: l2b.beam_search(a, t[5], 5, [bm[0], None], 4), -1),
            (lambda: l2b.beam_search(a, t[5], 5, [bm[0], a], 4), -1),
            (lambda: l2b.beam_search(a, t[5], 5, [bm[0], other], 4), -1),
            (lambda: l2b.beam_search(a, V, 5, bm, 4), -1),
            (lambda: l2b.beam_search(a, -1, 5, bm, 4), -1),
            (lambda: l2b.beam_search(a, t[5], -1, bm, 4), -1),
            (lambda: l2b.beam_search(a, t[5], S, bm, 4), -1),
            (lambda: l2b.beam_search(a, t[5], 5, bm, -1), -1),
            (lambda: l2b.beam_search(a, t[5], 71, bm, 4), -7),
            (lambda: l2b.beam_search(pr.b, t[5], 5, pr.scratch, 4), -2),
        ]
        for i, (call, status) in enumerate(bad):
            with pytest.raises(l2b.L2BError) as e:
                call()
            assert e.value.status == status, (i, e.value.status)
        # n_steps == 0 runs and changes nothing
        l2b.fork(a, bm[:1], 20)
        toks, lps, ran = l2b.beam_search(a, t[5], 5, bm, 0)
        assert ran == 0 and all(len(x) == 0 for x in toks) and not lps.any()
        assert pages_held(bm[0]) == 1 and pages_held(bm[1]) == 0
        other.close()
    finally:
        pr.close()
    # 2B > vocab_size: a 3-token vocabulary admits one beam, not two
    from llama2_zig_b200.checkpoint import shape_checkpoint
    with l2b.Transformer(shape_checkpoint((32, 64, 1, 4, 2, 3, 64)), synthetic_seed=1, kv_layout="paged") as m:
        s = [m.session(), m.session()]
        with pytest.raises(l2b.L2BError) as e:
            l2b.beam_search(m, 0, 0, s, 2)
        assert e.value.status == -1
        toks, lps, ran = l2b.beam_search(m, 0, 0, s[:1], 2, stop_on_bos=False)
        assert ran == 2 and len(toks[0]) == 2
        for x in s:
            x.close()


# ---- 5: the demo ----------------------------------------------------------------------------------------

def test_demo_beam(l2b, stories15m, tokenizer_path):  # noqa: F811
    exe = os.path.join(ROOT, "llama2.zig_b200", "bin", "llama2_b200")
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    with l2b.Transformer(ck, kv_layout="paged") as m:
        beams = [m.session() for _ in range(3)]
        toks, lps, _ = l2b.beam_search(m, 1, 0, beams, 48)
        for b in beams:
            b.close()
    want = demo_text(tokenizer_path, toks[0])
    assert len(want) > 0
    r = subprocess.run([exe, stories15m, "-n", "48", "-z", tokenizer_path, "--beam", "3", "-v"], capture_output=True,
                       check=True, timeout=300)
    assert r.stdout.rstrip(b"\n") == want.rstrip(b"\n")
    results = [ln for ln in r.stderr.decode().splitlines() if ln.startswith("result ")]
    assert len(results) == 3 and f"log-probability {lps[0]:g}" in results[0], results


# ---- 6: llama2-7B -----------------------------------------------------------------------------------------

@pytest.mark.slow
def test_llama2_7b(l2b):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint("llama2-7B")
    ck.seq_len = 2048
    n_prompt, n_beams = 1984, 4
    toks = teacher_tokens(n_prompt + 1, ck.vocab_size)
    with l2b.Transformer(ck, synthetic_seed=7, weight_format="bf16", kv_format="bf16", kv_layout="paged") as a, \
            l2b.Transformer(ck, synthetic_seed=7, weight_format="bf16", kv_format="bf16") as b:
        a.prefill(toks[:n_prompt], want_logits=False)
        b.prefill(toks[:n_prompt], want_logits=False)
        beams = [a.session() for _ in range(n_beams)]
        scratch = [b.session() for _ in range(n_beams)]
        try:
            got = l2b.beam_search(a, toks[n_prompt], n_prompt, beams, 16, stop_on_bos=False)
            ms, _ = a.last_timing()
            cands = twin_cands(l2b, b, scratch, toks[n_prompt], n_prompt, 2 * n_beams)
            want = ref_search(cands, toks[n_prompt], n_beams, 16, False)
            assert got[2] == want[2] == 16
            for x, y in zip(got[0], want[0]):
                _eq(x, y, "llama2-7B tokens")
            _eq(got[1], want[1], "llama2-7B logprobs")
            info = a.kv_pool_info()
            print(f"llama2-7B beam search B={n_beams}, 16 steps from {n_prompt}: {ms:.1f} ms, "
                  f"pages in use {info['pages_in_use']} (src {pages_held(a)}), "
                  f"beams hold {[pages_held(x) for x in beams]}")
            assert info["pages_in_use"] <= pages_held(a) + n_beams
        finally:
            for s in beams + scratch:
                s.close()
