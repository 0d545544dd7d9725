#!/usr/bin/env python
"""Greedy speculative decoding on llama2-7B (l2b_verify_argmax_ragged, l2b_generate_speculative).

  python scripts/bench_speculative.py [--repeats 2] [--tokens 64]

One llama2-7B model with synthetic fp32 weights (seed 7, as bench.py) and sessions on it, all after the same
8-token prompt.  G is the known greedy stream of --tokens tokens from there (generate_argmax_batch, n = 1).

Arms, alternated within each repeat (the first repeat warms every shape up and is not printed):
  generate_argmax        l2b_generate_argmax of --tokens tokens: the fastest single stream;
  generate_argmax_batch  l2b_generate_argmax_batch of one session: the bit-identical reference;
  verify k, alpha        rounds of l2b_verify_argmax_ragged over G: each round's kk = min(k, left - 1) drafts
                         are G's next tokens, each replaced by another token with seeded probability
                         1 - alpha; the round emits n_accept + 1 tokens, which must be G's.  k in {1, 2, 3,
                         7}, alpha in {1, 0.9, 0.7, 0.5, 0}.  Reported against the expected tokens per round
                         (1 - alpha^(k+1)) / (1 - alpha) (k + 1 at alpha = 1), with the device time per
                         emitted token over generate_argmax's;
  early exit             one verify run of 4, 8 and 12 vectors (1, 2, 3 passes) rejected at its first draft,
                         and of 8 accepted: what a pass skipped after CTL_DONE costs (median of 5 calls);
  speculative            l2b_generate_speculative with a stories15M-shaped draft (seq_len 2048, seed 10),
                         k in {1, 3}: on unrelated synthetic weights its acceptance is near 0, so this
                         measures the draft round's overhead.
Device time is l2b_last_timing (CUDA events; for the verify arm the sum over its rounds), wall time a host
clock around calls that end in a synchronise.  The break-even alpha of each k is where the verify arm's
device time per token, linearly interpolated between the measured alphas, crosses generate_argmax's.
One JSON line per measurement; the card's name, power limit and maximum SM clock (read-only nvidia-smi
query) are printed in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPE = (4096, 11008, 32, 32, 32, -32000, 2048)     # llama2-7B, unshared classifier
DRAFT_SHAPE = (288, 768, 6, 6, 6, 32000, 2048)      # stories15M layers, llama2-7B's context
SEED, DRAFT_SEED = 7, 10
KS = [1, 2, 3, 7]
ALPHAS = [1.0, 0.9, 0.7, 0.5, 0.0]


def teacher(b, n, vocab):
    return [(1 + 7919 * p + 104729 * b) % vocab for p in range(n)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def expected_per_round(alpha, k):
    return float(k + 1) if alpha == 1.0 else (1.0 - alpha ** (k + 1)) / (1.0 - alpha)


def verify_rounds(l2b, t, first, p, g, k, alpha, rng, V):
    """Rounds of verify over the known stream g from (first, p).  Returns (device ms, wall ms, rounds,
    [(vectors, ms)] per round)."""
    n, done, dev, per = len(g), 0, 0.0, []
    t0 = time.perf_counter()
    while done < n:
        kk = min(k, n - done - 1)
        d = [int(x) for x in g[done:done + kk]]
        for j in range(kk):
            if rng.random() >= alpha:
                d[j] = (d[j] + 1 + int(rng.integers(V - 1))) % V
        tok = first if done == 0 else int(g[done - 1])
        got, acc = l2b.verify_argmax_ragged([t], [[tok] + d], [p + done])
        ms = t.last_timing()[0]
        dev += ms
        per.append((kk + 1, ms))
        a = int(acc[0])
        assert got[0].tolist() == g[done:done + a + 1].tolist(), "verify left the greedy stream"
        done += a + 1
    return dev, (time.perf_counter() - t0) * 1e3, len(per), per


def break_even(alphas, per_token, t1):
    """The alpha where per_token(alpha) crosses t1, linearly interpolated; None if it does not cross."""
    pts = sorted(zip(alphas, per_token))
    for (a0, y0), (a1, y1) in zip(pts, pts[1:]):
        if (y0 - t1) * (y1 - t1) <= 0 and y0 != y1:
            return a0 + (t1 - y0) * (a1 - a0) / (y1 - y0)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--tokens", type=int, default=64)
    args = ap.parse_args()

    import torch
    import llama2_zig_b200 as l2b
    from llama2_zig_b200.checkpoint import shape_checkpoint

    if not torch.cuda.is_available():
        sys.exit("bench_speculative.py needs a GPU")
    print(json.dumps({"card": card()}), flush=True)

    ck = shape_checkpoint(SHAPE)
    V, N = ck.vocab_size, args.tokens
    prompt = teacher(3, 9, V)
    p, first = len(prompt) - 1, prompt[-1]
    m = l2b.Transformer(ck, synthetic_seed=SEED)
    t = m.session()
    draft = l2b.Transformer(shape_checkpoint(DRAFT_SHAPE), synthetic_seed=DRAFT_SEED)
    for s in (m, t, draft):
        s.prefill(prompt[:-1], 0, want_logits=False)
    g = l2b.generate_argmax_batch([m], [first], [p], N, stop_on_bos=False)[0]
    assert len(g) == N

    for r in range(args.repeats + 1):
        show = r > 0
        rng = np.random.default_rng(1000 + r)
        # ---- yardsticks
        base = {}
        for arm in ("generate_argmax", "generate_argmax_batch"):
            t0 = time.perf_counter()
            if arm == "generate_argmax":
                out = m.generate_argmax(first, p, N, stop_on_bos=False)
            else:
                out = l2b.generate_argmax_batch([m], [first], [p], N, stop_on_bos=False)[0]
            wall = (time.perf_counter() - t0) * 1e3
            dev = m.last_timing()[0]
            assert out.tolist() == g.tolist(), arm
            base[arm] = dev / N
            if show:
                print(json.dumps({"what": "yardstick", "arm": arm, "repeat": r, "tokens": N,
                                  "device_ms": round(dev, 2), "wall_ms": round(wall, 2),
                                  "device_tok_s": round(N / dev * 1e3, 2), "wall_tok_s": round(N / wall * 1e3, 2)}),
                      flush=True)
        t1 = base["generate_argmax"]
        # ---- verify rounds over the known stream
        per_vec = {}
        per_token = {k: [] for k in KS}
        for k in KS:
            for alpha in ALPHAS:
                dev, wall, rounds, per = verify_rounds(l2b, t, first, p, g, k, alpha, rng, V)
                per_token[k].append(dev / N)
                if alpha == 0.0 or alpha == 1.0:
                    for nv, ms in per:
                        per_vec.setdefault((nv, "rejected at 1" if alpha == 0.0 else "accepted"), []).append(ms)
                if show:
                    print(json.dumps({"what": "verify", "repeat": r, "k": k, "alpha": alpha, "tokens": N,
                                      "rounds": rounds, "tokens_per_round": round(N / rounds, 3),
                                      "expected_tokens_per_round": round(expected_per_round(alpha, k), 3),
                                      "device_ms": round(dev, 2), "wall_ms": round(wall, 2),
                                      "device_tok_s": round(N / dev * 1e3, 2), "wall_tok_s": round(N / wall * 1e3, 2),
                                      "device_ms_per_token_over_generate_argmax": round(dev / N / t1, 3)}),
                          flush=True)
        if show:
            for (nv, how), ms in sorted(per_vec.items()):
                print(json.dumps({"what": "verify_round_ms", "repeat": r, "vectors": nv, "drafts": how,
                                  "rounds": len(ms), "median_ms": round(float(np.median(ms)), 3)}), flush=True)
            for k in KS:
                be = break_even(ALPHAS, per_token[k], t1)
                print(json.dumps({"what": "break_even_alpha", "repeat": r, "k": k,
                                  "alpha": None if be is None else round(be, 3)}), flush=True)
        # ---- early exit: runs rejected at their first draft, 1 .. 3 passes, against 2 full passes
        cost = {}
        for nv, how in ((4, "rejected"), (8, "rejected"), (12, "rejected"), (8, "accepted")):
            run = [first] + [int(x) for x in g[:nv - 1]]
            if how == "rejected":
                run[1] = (run[1] + 1) % V
            ms = []
            for _ in range(5):
                _, acc = l2b.verify_argmax_ragged([t], [run], [p])
                assert int(acc[0]) == (0 if how == "rejected" else nv - 1)
                ms.append(t.last_timing()[0])
            cost[(nv, how)] = float(np.median(ms))
            if show:
                print(json.dumps({"what": "early_exit", "repeat": r, "vectors": nv, "passes": (nv + 3) // 4,
                                  "drafts": how, "median_ms": round(cost[(nv, how)], 3)}), flush=True)
        if show:
            one = cost[(4, "rejected")]
            print(json.dumps({"what": "early_exit_summary", "repeat": r,
                              "skipped_pass_ms": round(cost[(8, "rejected")] - one, 3),
                              "two_pass_over_one_pass_rejected_at_1": round(cost[(8, "rejected")] / one, 3),
                              "three_pass_over_one_pass_rejected_at_1": round(cost[(12, "rejected")] / one, 3),
                              "full_second_pass_ms": round(cost[(8, "accepted")] - one, 3)}), flush=True)
        # ---- a real draft
        for k in (1, 3):
            draft.reset()
            draft.prefill(prompt[:-1], 0, want_logits=False)
            t0 = time.perf_counter()
            out, rounds = m.generate_speculative(draft, first, p, N, k, stop_on_bos=False)
            wall = (time.perf_counter() - t0) * 1e3
            dev = m.last_timing()[0]
            assert out.tolist() == g.tolist(), "generate_speculative left the greedy stream"
            if show:
                print(json.dumps({"what": "speculative", "draft": "stories15M-shaped, seed 10", "repeat": r, "k": k,
                                  "tokens": N, "rounds": rounds, "tokens_per_round": round(N / rounds, 3),
                                  "device_ms": round(dev, 2), "wall_ms": round(wall, 2),
                                  "device_tok_s": round(N / dev * 1e3, 2), "wall_tok_s": round(N / wall * 1e3, 2),
                                  "device_ms_per_token_over_generate_argmax": round(dev / N / t1, 3)}), flush=True)
    for s in (t, draft, m):
        s.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
