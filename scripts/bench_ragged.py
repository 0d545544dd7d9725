#!/usr/bin/env python
"""Admitting a prompt into running decode sessions, and packing short prompts, on one llama2-7B model
(l2b_forward_ragged / l2b_forward_argmax_ragged against l2b_prefill + the *_batch calls).

  python scripts/bench_ragged.py [--decoders 1,2,3] [--prompt 256] [--new 64] [--arrive 16] [--repeats 2]

One model with synthetic fp32 weights (seed 7, as bench.py) and sessions on it.

Admission.  D sessions decode with their teacher tokens forced (session b: teacher(b)).  At step
--arrive a new session brings a --prompt-token prompt.  Two arms, from the same state:
  stall   l2b_prefill of the prompt but its last token (no logits), then l2b_forward_argmax_batch of
          the D + 1 sessions (the new one starts with its prompt's last token);
  ragged  each call gives every decoder 1 token and fills the other 4 - D slots of the pass with the
          prompt's next tokens (l2b_forward_argmax_ragged); once the prompt is in, the new session
          decodes 1 token per call next to the decoders.
A decoder leaves after --new tokens past the arrival; once no decoder is left, the rest of a prompt
goes in one call.  Reported per arm, from the arrival on, in device time (each call's CUDA events,
l2b_last_timing, summed): the new session's time to first token; the longest gap between two
consecutive tokens of any decoder (the calls in between included); the total until every session has
--new new tokens; and the aggregate rate of those (D + 1) x --new tokens.

Packing.  Prompts of 5, 6, 7 and 9 tokens on 4 fresh sessions: 4 l2b_prefill calls with logits (each
ends in a single decode step) against one l2b_forward_ragged call.  Passes over the weights are counted
from the shapes; time is a host clock around the calls (each ends in a synchronise; l2b_prefill's own
events do not cover its final single step), median of --pack-repeats.

The arms alternate within each repeat; the first repeat warms every shape up and is not printed.  One
JSON line per measurement; the card's name and power limit (read-only nvidia-smi query) are printed in
the same run.
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
PACK = [5, 6, 7, 9]


def teacher(b, n, vocab):
    return [(1 + 7919 * p + 104729 * b) % vocab for p in range(n)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def admission(l2b, dec, p, toks, prompt, arrive, new, ragged):
    """One arm from a fresh state.  Returns (ttft_ms, max_gap_ms, total_ms, calls)."""
    D = len(dec)
    for s in dec + [p]:
        s.reset()
    for i in range(arrive):                                      # the decoders before the arrival
        l2b.forward_argmax_batch(dec, [toks[b][i] for b in range(D)], [i] * D)
    got = [0] * D                                                # decoders' tokens since the arrival
    since = [0.0] * D                                            # device ms since a decoder's last token
    gap, total, ttft, calls = 0.0, 0.0, None, 0
    done, p_new = 0, 0                                           # prompt tokens in, new session's tokens

    def account(ms, produced):
        nonlocal gap, total
        total += ms
        for b in range(D):
            since[b] += ms
            if produced[b]:
                gap = max(gap, since[b])
                since[b] = 0.0
                got[b] += 1

    if not ragged:
        p.prefill(prompt[:-1], 0, want_logits=False)
        account(p.last_timing()[0], [False] * D)
        calls += 1
        done = len(prompt) - 1
    while p_new < new or min(got) < new:
        live = [b for b in range(D) if got[b] < new]
        sess = [dec[b] for b in live]
        pos = [arrive + got[b] for b in live]
        runs = [[toks[b][q]] for b, q in zip(live, pos)]
        if done < len(prompt):                                   # the prompt's next tokens fill the pass
            c = len(prompt) - done if not live else min(4 - len(live), len(prompt) - done)
            runs.append(prompt[done:done + c])
            pos.append(done)
            done += c
            p_out = done == len(prompt)                          # the prompt's last token: the first output
        else:                                                    # the new session decodes
            runs.append([toks[D][len(prompt) + p_new - 1]])
            pos.append(len(prompt) + p_new - 1)
            p_out = True
        sess.append(p)
        if ragged:
            l2b.forward_argmax_ragged(sess, runs, pos)
        else:
            assert all(len(r) == 1 for r in runs)
            l2b.forward_argmax_batch(sess, [r[0] for r in runs], pos)
        account(sess[0].last_timing()[0], [b in live for b in range(D)])
        calls += 1
        if p_out:
            p_new += 1
            if ttft is None:
                ttft = total
    return ttft, gap, total, calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--decoders", default="1,2,3")
    ap.add_argument("--prompt", type=int, default=256)
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--arrive", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--pack-repeats", type=int, default=11)
    args = ap.parse_args()

    import torch
    import llama2_zig_b200 as l2b
    from llama2_zig_b200.checkpoint import shape_checkpoint

    if not torch.cuda.is_available():
        sys.exit("bench_ragged.py needs a GPU")
    print(json.dumps({"card": card()}), flush=True)

    ck = shape_checkpoint(SHAPE)
    V = ck.vocab_size
    m = l2b.Transformer(ck, synthetic_seed=SEED)
    sess = [m] + [m.session() for _ in range(3)]
    n_tok = args.arrive + args.new + args.prompt + 1
    toks = [teacher(b, n_tok, V) for b in range(4)]

    for D in [int(x) for x in args.decoders.split(",")]:
        dec, p = sess[:D], sess[D]
        prompt = teacher(100 + D, args.prompt, V)
        for r in range(args.repeats + 1):
            for arm in ("stall", "ragged"):
                ttft, gap, total, calls = admission(l2b, dec, p, toks[:D] + [toks[3]], prompt, args.arrive, args.new,
                                                    arm == "ragged")
                if r:
                    print(json.dumps({"what": "admission", "arm": arm, "decoders": D, "prompt": args.prompt,
                                      "new_tokens": args.new, "calls": calls, "ttft_ms": round(ttft, 2),
                                      "max_decoder_gap_ms": round(gap, 2), "total_ms": round(total, 2),
                                      "tok_s": round((D + 1) * args.new / (total / 1e3), 2)}), flush=True)

    prompts = [teacher(200 + i, k, V) for i, k in enumerate(PACK)]
    passes_prefill = sum((k - 2) // 4 + 1 for k in PACK)          # l2b_prefill's batched groups of k - 1 tokens
    passes_ragged = (sum(PACK) + 3) // 4
    for r in range(2):
        times = {"prefill": [], "ragged": []}
        for _ in range(args.pack_repeats):
            for arm in ("prefill", "ragged"):
                for s in sess:
                    s.reset()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if arm == "prefill":
                    for s, pr in zip(sess, prompts):
                        s.prefill(pr, 0, want_logits=True)
                else:
                    l2b.forward_ragged(sess, prompts, [0] * 4)
                times[arm].append((time.perf_counter() - t0) * 1e3)
                if arm == "ragged":
                    dev = m.last_timing()
        if r:
            print(json.dumps({"what": "packing", "arm": "4 x l2b_prefill", "prompts": PACK,
                              "passes": f"{passes_prefill} batched + 4 single steps",
                              "wall_ms_median": round(float(np.median(times["prefill"])), 2)}), flush=True)
            print(json.dumps({"what": "packing", "arm": "1 x l2b_forward_ragged", "prompts": PACK,
                              "passes": passes_ragged, "launches": dev[1], "device_ms": round(dev[0], 2),
                              "wall_ms_median": round(float(np.median(times["ragged"])), 2)}), flush=True)
    for s in sess[1:]:
        s.close()
    m.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
