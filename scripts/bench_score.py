#!/usr/bin/env python
"""Scoring rate of a known sequence (l2b_score: per-position log-probabilities, teacher forcing).

  python scripts/bench_score.py [--tokens 256] [--repeats 3]

llama2-7B with synthetic fp32 weights (seed 7, as bench.py), --tokens teacher tokens scored from position
0 (tokens - 1 positions) on the batched path, against:
  * l2b_prefill of the same tokens - 1 positions (logits-free: the rate scoring can approach);
  * a host loop of l2b_forward with a NumPy float64 log-softmax per position (wall time: single steps
    carry no events by default).
The stories15M and stories110M shapes (synthetic weights, whole context) score on the device loop
G_SCORE_LOOP, against l2b_generate_argmax over the same positions with the same tokens forced.
Device times are the library's own CUDA events around each call (l2b_last_timing); a host clock around
each call (every call ends in a synchronise) gives the wall time.  The L2 cache is flushed (256 MiB
memset) before each timed call, the first repeat only warms up, and the variants alternate within each
repeat.  One JSON line per measurement; the card's name and power limit (read-only nvidia-smi query)
are printed in the same run.
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

SEED = 7


def teacher(n, vocab):
    return [(1 + 7919 * p) % vocab for p in range(n)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def log_softmax_at(logits, target):
    x = logits.astype(np.float64)
    m = x.max()
    return (x[target] - m) - np.log(np.sum(np.exp(x - m)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import torch
    import llama2_zig_b200 as l2b
    from llama2_zig_b200.checkpoint import shape_checkpoint

    if not torch.cuda.is_available():
        sys.exit("bench_score.py needs a GPU")
    print(json.dumps({"card": card()}), flush=True)
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def flush():
        scratch.zero_()
        torch.cuda.synchronize()

    def timed(fn):
        flush()
        t0 = time.perf_counter()
        fn()
        return time.perf_counter() - t0

    def report(r, model, what, n, ms=None, wall=None, launches=None):
        if not r:
            return
        rec = {"model": model, "what": what, "positions": n}
        if ms is not None:
            rec.update(device_ms=round(ms, 2), tok_s=round(n / (ms / 1e3), 1))
        if wall is not None:
            rec.update(wall_ms=round(wall * 1e3, 2), wall_tok_s=round(n / wall, 1))
        if launches is not None:
            rec["launches"] = launches
        print(json.dumps(rec), flush=True)

    # llama2-7B: the batched path
    ck = shape_checkpoint("llama2-7B")
    toks = teacher(args.tokens, ck.vocab_size)
    n = len(toks) - 1
    with l2b.Transformer(ck, synthetic_seed=SEED) as m:
        for r in range(args.repeats + 1):
            m.reset()
            wall = timed(lambda: m.score(toks, 0))
            ms, launches = m.last_timing()
            report(r, "llama2-7B", "l2b_score", n, ms, wall, launches)
            m.reset()
            wall = timed(lambda: m.prefill(toks[:-1], 0, want_logits=False))
            ms, launches = m.last_timing()
            report(r, "llama2-7B", "l2b_prefill", n, ms, wall, launches)
            m.reset()
            out = np.empty(ck.vocab_size, np.float32)

            def host_loop():
                for i in range(n):
                    m.forward_into(toks[i], i, out)
                    log_softmax_at(out, toks[i + 1])
            wall = timed(host_loop)
            report(r, "llama2-7B", "host loop of l2b_forward + NumPy log-softmax", n, None, wall)

    # small models: the device loop
    for name in ("stories15M", "stories110M"):
        ck = shape_checkpoint(name)
        toks = teacher(min(args.tokens, ck.seq_len + 1), ck.vocab_size)
        n = len(toks) - 1
        with l2b.Transformer(ck, synthetic_seed=SEED) as m:
            for r in range(args.repeats + 1):
                m.reset()
                wall = timed(lambda: m.score(toks, 0))
                ms, launches = m.last_timing()
                report(r, name, "l2b_score", n, ms, wall, launches)
                m.reset()
                wall = timed(lambda: m.generate_argmax(toks[0], 0, n, forced=toks[1:], stop_on_bos=False))
                ms, launches = m.last_timing()
                report(r, name, "l2b_generate_argmax", n, ms, wall, launches)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
