#!/usr/bin/env python
"""Forking sessions from a shared prompt on one llama2-7B model (l2b_fork).

  python scripts/bench_fork.py [--repeats 2] [--iters 5] [--prompt 256]

One model with synthetic fp32 weights (seed 7, as bench.py) and 7 sessions on it.

Copy rate.  The model's own context holds 2048 positions; l2b_fork copies rows [0, n_pos) of its key and
value caches into n_dst sessions, for n_pos in {256, 1024, 2048} and n_dst in {1, 3, 7}.  Device time is
l2b_last_timing (CUDA events around the call's launches), the median of --iters calls.  The fork reads the
source once and writes it n_dst times: bytes = (1 + n_dst) * 2 * L * n_pos * kv_dim * 4, and the
bytes-bound share is those bytes over the time over 3.35 TB/s (the H100 SXM data sheet's HBM3 rate).
The yardstick, in the same run: torch `copy_` of the same slices between one source pair and one
destination pair of (L, seq_len, kv_dim) tensors, once per destination and per cache (2 * n_dst copies,
each reading and writing its slice), timed with CUDA events, median of --iters.

Best of 4 from a --prompt-token prompt: time to the four first-token distributions (temperature 1,
top-p 0.9).  Two arms:
  ragged  l2b_forward_sample_ragged of the whole prompt on 4 fresh sessions (4 x prompt vectors, 4 per
          weight pass);
  fork    l2b_prefill of prompt[:-1] on one session, l2b_fork to 3 more, then one
          l2b_forward_sample_batch of the last prompt token on all 4.
Both arms must give bit-identical probabilities and candidates.  Reported: device time (the sum of each
call's l2b_last_timing) and host wall time (a host clock around the calls, which end in a synchronise).

The arms alternate within each repeat; the first repeat warms every shape up and is not printed.  One
JSON line per measurement; the card's name, power limit and maximum SM clock (read-only nvidia-smi query)
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

SHAPE = (4096, 11008, 32, 32, 32, -32000, 2048)     # llama2-7B, unshared classifier
SEED = 7
HBM_BYTES_S = 3.35e12                               # H100 SXM data sheet
N_POS = [256, 1024, 2048]
N_DST = [1, 3, 7]


def teacher(b, n, vocab):
    return [(1 + 7919 * p + 104729 * b) % vocab for p in range(n)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def time_fork(l2b, m, dsts, n_pos, iters):
    ms = []
    for _ in range(iters):
        l2b.fork(m, dsts, n_pos)
        t, launches = m.last_timing()
        ms.append(t)
    return float(np.median(ms)), launches


def time_torch(torch, src, dst, n_dst, n_pos, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(iters):
        e0.record()
        for _ in range(n_dst):
            for s, d in zip(src, dst):
                d[:, :n_pos].copy_(s[:, :n_pos])
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def best_of_4(l2b, sess, prompt, arm, temp, top_p):
    """One arm from fresh sessions.  Returns ((probs, candidates, n_cand), device_ms, wall_ms)."""
    for s in sess:
        s.reset()
    P = len(prompt)
    t0 = time.perf_counter()
    if arm == "ragged":
        out = l2b.forward_sample_ragged(sess, [prompt] * 4, [0] * 4, temp, top_p)
        dev = sess[0].last_timing()[0]
    else:
        sess[0].prefill(prompt[:-1], 0, want_logits=False)
        dev = sess[0].last_timing()[0]
        l2b.fork(sess[0], sess[1:], P - 1)
        dev += sess[0].last_timing()[0]
        out = l2b.forward_sample_batch(sess, [prompt[-1]] * 4, [P - 1] * 4, temp, top_p)
        dev += sess[0].last_timing()[0]
    wall = (time.perf_counter() - t0) * 1e3
    return out, dev, wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--prompt", type=int, default=256)
    args = ap.parse_args()

    import torch
    import llama2_zig_b200 as l2b
    from llama2_zig_b200.checkpoint import shape_checkpoint

    if not torch.cuda.is_available():
        sys.exit("bench_fork.py needs a GPU")
    print(json.dumps({"card": card()}), flush=True)

    ck = shape_checkpoint(SHAPE)
    V, L, S = ck.vocab_size, ck.n_layers, ck.seq_len
    kv = ck.dim * ck.n_kv_heads // ck.n_heads
    m = l2b.Transformer(ck, synthetic_seed=SEED)
    sess = [m.session() for _ in range(7)]
    m.prefill(teacher(0, S, V), 0, want_logits=False)
    src = [torch.randn(L, S, kv, device="cuda") for _ in range(2)]
    dst = [torch.empty(L, S, kv, device="cuda") for _ in range(2)]

    for r in range(args.repeats + 1):
        for n_pos in N_POS:
            for n_dst in N_DST:
                for arm in ("l2b_fork", "torch copy_"):
                    if arm == "l2b_fork":
                        ms, launches = time_fork(l2b, m, sess[:n_dst], n_pos, args.iters)
                        nbytes = (1 + n_dst) * 2 * L * n_pos * kv * 4
                    else:
                        ms, launches = time_torch(torch, src, dst, n_dst, n_pos, args.iters), 2 * n_dst
                        nbytes = 2 * n_dst * 2 * L * n_pos * kv * 4
                    if r:
                        gbs = nbytes / (ms * 1e-3) / 1e9
                        print(json.dumps({"what": "copy", "arm": arm, "repeat": r, "n_pos": n_pos, "n_dst": n_dst,
                                          "launches": launches, "device_ms": round(ms, 4), "bytes": nbytes,
                                          "GB_s": round(gbs, 1),
                                          "bytes_bound_share_of_3.35TB_s": round(gbs * 1e9 / HBM_BYTES_S, 3)}),
                              flush=True)

    prompt = teacher(100, args.prompt, V)
    temp, top_p = [1.0] * 4, [0.9] * 4
    four = sess[:4]
    for r in range(args.repeats + 1):
        outs = {}
        for arm in ("ragged", "fork"):
            outs[arm], dev, wall = best_of_4(l2b, four, prompt, arm, temp, top_p)
            passes = args.prompt if arm == "ragged" else f"{(args.prompt + 2) // 4} + 1 + the copy"
            if r:
                print(json.dumps({"what": "best_of_4", "arm": arm, "repeat": r, "prompt": args.prompt,
                                  "weight_passes": passes, "device_ms": round(dev, 2), "wall_ms": round(wall, 2)}),
                      flush=True)
        (pa, ca, ka), (pb, cb, kb) = outs["ragged"], outs["fork"]
        assert np.array_equal(pa, pb) and np.array_equal(ka, kb), "the arms' probabilities differ"
        for x, y in zip(ca, cb):
            assert (x is None) == (y is None) and (x is None or np.array_equal(x, y)), "the arms' candidates differ"
    print(json.dumps({"what": "best_of_4", "bit_identical": True}), flush=True)
    for s in sess:
        s.close()
    m.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
