#!/usr/bin/env python
"""Aggregate decode rate of n sessions on one llama2-7B model (l2b_create_session + l2b_forward_argmax_batch /
l2b_generate_argmax_batch / l2b_forward_sample_batch).

  python scripts/bench_sessions.py [--sessions 1,2,4,8] [--positions 256] [--warmup 4] [--repeats 2]

One model with synthetic fp32 weights (seed 7, as bench.py) and n-1 sessions on it.  Session b is
prefilled to 61*b positions (staggered, so the sessions' attention lengths differ), warmed up for
--warmup batched steps, and then teacher-forced over --positions positions through
l2b_forward_argmax_batch, one call per position ("batched step"), and in the same repeat through one
l2b_generate_argmax_batch call over the same positions with the teacher tokens forced ("device loop":
no host round trip per position).  A third run in the same repeat samples at the reference CLI's
defaults (temperature 1.0, top-p 0.9) through l2b_forward_sample_batch, one call per position
("sampled batched step"): each session's token is drawn on the host from its candidates with its own
seeded generator and fed back.  The three alternate within each repeat.  The L2 cache is flushed (256 MiB memset) before
each timed run.  Per call the library brackets its work with CUDA events (l2b_last_timing); the device
time of a run is their sum, and a host clock around the run (every call ends in a synchronise) gives
the wall time (the device loop is one call).  The single-stream references are the on-device loop of one context
(l2b_generate_argmax, bench.py's headline), timed the same way, and a host loop of l2b_forward_sample on
one context with the same draw (wall time only: single steps carry no events by default).  One JSON
line per measurement; the card's name and power limit (read-only nvidia-smi query) are printed in the
same run.
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
SEED = 7
TEMPERATURE, TOP_P = 1.0, 0.9                        # the reference CLI's defaults


def teacher(b, n, vocab):
    return [(1 + 7919 * p + 104729 * b) % vocab for p in range(n)]


def draw(rng, probs, cand, n_cand):
    """The host's part of top-p sampling: the candidates (or, when more passed than the device returned,
    the host's own filter of probs) sorted by probability, cut where the cumulative probability passes
    TOP_P, and one uniform draw walked along their CDF."""
    if n_cand < 0:
        idx = np.nonzero(probs >= np.float32((1.0 - TOP_P) / (probs.size - 1)))[0]
        pr = probs[idx]
    else:
        idx, pr = cand["index"], cand["prob"]
    order = np.argsort(-pr, kind="stable")
    idx, pr = idx[order], pr[order]
    cdf = np.cumsum(pr, dtype=np.float64)
    last = min(int(np.searchsorted(cdf, TOP_P, side="right")), idx.size - 1)
    return int(idx[min(int(np.searchsorted(cdf[:last + 1], rng.random() * cdf[last], side="right")), last)])


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="1,2,4,8")
    ap.add_argument("--positions", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    counts = [int(x) for x in args.sessions.split(",")]

    import torch
    import llama2_zig_b200 as l2b
    from llama2_zig_b200.checkpoint import shape_checkpoint

    if not torch.cuda.is_available():
        sys.exit("bench_sessions.py needs a GPU")
    print(json.dumps({"card": card()}), flush=True)
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def flush():
        scratch.zero_()
        torch.cuda.synchronize()

    ck = shape_checkpoint(SHAPE)
    V = ck.vocab_size
    m = l2b.Transformer(ck, synthetic_seed=SEED)
    sess = [m] + [m.session() for _ in range(max(counts) - 1)]
    P, W = args.positions, args.warmup
    starts = [61 * b for b in range(max(counts))]
    assert starts[-1] + W + P <= ck.seq_len
    toks = [teacher(b, starts[b] + W + P + 1, V) for b in range(len(sess))]

    # single stream: the on-device loop of one context over the same number of positions
    for r in range(args.repeats + 1):
        m.reset()
        flush()
        t0 = time.perf_counter()
        m.generate_argmax(toks[0][0], 0, P, forced=toks[0][1:P + 1], stop_on_bos=False)
        wall = time.perf_counter() - t0
        ms = m.last_timing()[0]
        if r:
            print(json.dumps({"what": "single-stream device loop", "positions": P, "device_ms": round(ms, 2),
                              "tok_s": round(P / (ms / 1e3), 2), "wall_tok_s": round(P / wall, 2)}), flush=True)
        # single stream, sampled: a host loop of forward_sample over the same number of positions
        m.reset()
        rng = np.random.default_rng(SEED)
        flush()
        t0 = time.perf_counter()
        tok = toks[0][0]
        for pos in range(P):
            probs, cand, k = m.forward_sample(tok, pos, TEMPERATURE, TOP_P, with_count=True)
            tok = draw(rng, probs, cand, k)
        wall = time.perf_counter() - t0
        if r:
            print(json.dumps({"what": "single-stream sampled steps", "positions": P,
                              "wall_tok_s": round(P / wall, 2)}), flush=True)

    for n in counts:
        group = sess[:n]
        def prepare(group):
            """Every session prefilled to its start and stepped --warmup positions."""
            for b, s in enumerate(group):
                s.reset()
                if starts[b]:
                    s.prefill(toks[b][:starts[b]], 0, want_logits=False)
            for i in range(W):
                pos = [starts[b] + i for b in range(n)]
                l2b.forward_argmax_batch(group, [toks[b][p] for b, p in enumerate(pos)], pos)

        for r in range(args.repeats + 1):                       # the first run warms every shape up
            prepare(group)
            flush()
            dev_ms, launches = 0.0, 0
            t0 = time.perf_counter()
            for i in range(W, W + P):
                pos = [starts[b] + i for b in range(n)]
                l2b.forward_argmax_batch(group, [toks[b][p] for b, p in enumerate(pos)], pos)
                ms, launches = group[0].last_timing()
                dev_ms += ms
            wall = time.perf_counter() - t0
            if r:
                print(json.dumps({"what": "batched step", "sessions": n, "positions": P,
                                  "launches_per_step": launches,
                                  "ms_per_step": round(dev_ms / P, 3),
                                  "tok_s": round(n * P / (dev_ms / 1e3), 2),
                                  "wall_tok_s": round(n * P / wall, 2)}), flush=True)
            # the same positions through the device loop, from the same state
            prepare(group)
            first = [toks[b][starts[b] + W] for b in range(n)]
            forced = [toks[b][starts[b] + W + 1:starts[b] + W + P + 1] for b in range(n)]
            flush()
            t0 = time.perf_counter()
            l2b.generate_argmax_batch(group, first, [starts[b] + W for b in range(n)], P, forced=forced,
                                      stop_on_bos=False)
            wall = time.perf_counter() - t0
            ms, launches = group[0].last_timing()
            if r:
                print(json.dumps({"what": "device loop", "sessions": n, "positions": P,
                                  "launches_per_step": launches // P,
                                  "ms_per_step": round(ms / P, 3),
                                  "tok_s": round(n * P / (ms / 1e3), 2),
                                  "wall_tok_s": round(n * P / wall, 2)}), flush=True)
            # the same positions sampled, each session's drawn token fed back, from the same state
            prepare(group)
            rngs = [np.random.default_rng(SEED + b) for b in range(n)]
            tok = [toks[b][starts[b] + W] for b in range(n)]
            flush()
            dev_ms = 0.0
            t0 = time.perf_counter()
            for i in range(W, W + P):
                pos = [starts[b] + i for b in range(n)]
                probs, cands, counts = l2b.forward_sample_batch(group, tok, pos, [TEMPERATURE] * n, [TOP_P] * n)
                ms, launches = group[0].last_timing()
                dev_ms += ms
                tok = [draw(rngs[b], probs[b], cands[b], counts[b]) for b in range(n)]
            wall = time.perf_counter() - t0
            if r:
                print(json.dumps({"what": "sampled batched step", "sessions": n, "positions": P,
                                  "launches_per_step": launches,
                                  "ms_per_step": round(dev_ms / P, 3),
                                  "tok_s": round(n * P / (dev_ms / 1e3), 2),
                                  "wall_tok_s": round(n * P / wall, 2)}), flush=True)
    for s in sess[1:]:
        s.close()
    m.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
