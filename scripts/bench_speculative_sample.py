#!/usr/bin/env python
"""Sampled speculative decoding on llama2-7B (l2b_verify_sample_ragged, l2h_generate_speculative_sample).

  python scripts/bench_speculative_sample.py [--repeats 2] [--tokens 32]

One llama2-7B model with synthetic fp32 weights (seed 7, as bench.py) and sessions on it, all after the same
8-token prompt, sampled at T = 1.0, top-p = 0.9 from seed 42.

Arms, alternated within each repeat (the first repeat warms every shape up and is not printed):
  plain        the reference loop: per token one l2b_forward_sample_batch of one session and the host twin's
               sampler (l2h_sample_top_p_candidates on the device's candidates).  Device time is the sum of
               the calls' l2b_last_timing;
  speculative  l2h_generate_speculative_sample with the target's own weights as draft (a session of the
               model: every proposal that the coins couple is accepted, but each proposal is a full llama2-7B
               step) at k = 1 and 3, and a stories15M-shaped draft (seq_len 2048, seed 10) at k = 1 and 3.
               The tokens must equal the plain arm's.  Wall time is a host clock around the call; the call
               does not report device time;
  verify round l2b_verify_sample_ragged of k + 1 positions (median of 5), the device time of one round's
               target work, against one plain step.
The acceptance rate is accepted drafts (tokens - rounds) over rounds * k; the last round may propose fewer
than k, so the rate is a lower bound.
D2H bytes per round are what the verify call copies: k + 1 positions of vocab_size probabilities and 8192
candidates, plus one count each.  One JSON line per measurement; the card's name, power limit and maximum
SM clock (read-only nvidia-smi query) are printed in the same run.
"""
import argparse
import ctypes as C
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
SEED, DRAFT_SEED, COIN_SEED = 7, 10, 42
T, TOP_P = 1.0, 0.9
FP = C.POINTER(C.c_float)
IP = C.POINTER(C.c_int32)


class PI(C.Structure):
    _fields_ = [("prob", C.c_float), ("index", C.c_int32)]


def teacher(b, n, vocab):
    return [(1 + 7919 * p + 104729 * b) % vocab for p in range(n)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def load_host(l2b):
    C.CDLL(l2b.lib_path(), mode=C.RTLD_GLOBAL)
    h = C.CDLL(os.path.join(ROOT, "llama2.zig_b200", "lib", "libllama2_host.so"))
    h.l2h_seed.argtypes = [C.c_uint64]
    h.l2h_sample.argtypes = [FP, C.c_int32]
    h.l2h_sample_top_p.argtypes = [FP, C.c_int32, C.c_float, C.c_void_p]
    h.l2h_sample_top_p_candidates.argtypes = [C.POINTER(PI), C.c_int32, C.c_float]
    cfg = C.POINTER(l2b.L2BConfig)
    h.l2h_generate_speculative_sample.argtypes = [C.c_void_p, cfg, C.c_void_p, cfg, C.c_int32, C.c_int32, C.c_int32,
                                                  C.c_int32, C.c_float, C.c_float, C.c_int32, IP, IP, IP]
    return h


def plain(l2b, h, t, first, p, n):
    """(tokens, device ms, wall ms) of the reference loop."""
    h.l2h_seed(COIN_SEED)
    out, dev, tok = [], 0.0, first
    t0 = time.perf_counter()
    for q in range(p, p + n):
        probs, cands, nc = l2b.forward_sample_batch([t], [tok], [q], [T], [TOP_P])
        dev += t.last_timing()[0]
        if nc[0] > 0:
            tok = h.l2h_sample_top_p_candidates((PI * int(nc[0])).from_buffer_copy(cands[0].tobytes()), int(nc[0]), TOP_P)
        else:
            tok = h.l2h_sample_top_p(probs[0].ctypes.data_as(FP), probs.shape[1], TOP_P, (C.c_uint64 * probs.shape[1])())
        out.append(tok)
    return out, dev, (time.perf_counter() - t0) * 1e3


def speculative(h, target, draft, first, p, n, k):
    h.l2h_seed(COIN_SEED)
    out = np.full(n, -1, dtype=np.int32)
    done, rounds = C.c_int32(), C.c_int32()
    t0 = time.perf_counter()
    rc = h.l2h_generate_speculative_sample(target.h, C.byref(target.cfg), draft.h, C.byref(draft.cfg), first, p, n, k,
                                           T, TOP_P, 0, out.ctypes.data_as(IP), C.byref(done), C.byref(rounds))
    wall = (time.perf_counter() - t0) * 1e3
    assert rc == 0, rc
    return out[:done.value].tolist(), rounds.value, wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--tokens", type=int, default=32)
    args = ap.parse_args()

    import torch
    import llama2_zig_b200 as l2b
    from llama2_zig_b200.checkpoint import shape_checkpoint

    if not torch.cuda.is_available():
        sys.exit("bench_speculative_sample.py needs a GPU")
    print(json.dumps({"card": card()}), flush=True)
    h = load_host(l2b)

    ck = shape_checkpoint(SHAPE)
    V, N = ck.vocab_size, args.tokens
    prompt = teacher(3, 9, V)
    p, first = len(prompt) - 1, prompt[-1]
    m = l2b.Transformer(ck, synthetic_seed=SEED)
    own, ref = m.session(), m.session()
    small = l2b.Transformer(shape_checkpoint(DRAFT_SHAPE), synthetic_seed=DRAFT_SEED)
    for s in (m, own, ref, small):
        s.prefill(prompt[:-1], 0, want_logits=False)
    d2h_per_pos = 4 * V + 8 * 8192 + 4

    for r in range(args.repeats + 1):
        show = r > 0
        want, dev, wall = plain(l2b, h, ref, first, p, N)
        base = dev / N
        if show:
            print(json.dumps({"what": "plain", "repeat": r, "tokens": N, "device_ms": round(dev, 2),
                              "wall_ms": round(wall, 2), "device_tok_s": round(N / dev * 1e3, 2),
                              "wall_tok_s": round(N / wall * 1e3, 2)}), flush=True)
        for name, draft in (("own weights", own), ("stories15M-shaped, seed 10", small)):
            for k in (1, 3):
                for s in (m, draft):
                    s.reset()
                    s.prefill(prompt[:-1], 0, want_logits=False)
                got, rounds, wall_s = speculative(h, m, draft, first, p, N, k)
                assert got == want, (name, k)
                # accepted drafts: each round emits its accepted drafts plus the target's own token
                accepted = len(got) - rounds
                if show:
                    print(json.dumps({"what": "speculative", "draft": name, "repeat": r, "k": k, "tokens": len(got),
                                      "rounds": rounds, "tokens_per_round": round(len(got) / rounds, 3),
                                      "accepted_drafts": accepted,
                                      "acceptance_at_least": round(accepted / max(1, rounds * k), 3),
                                      "wall_ms": round(wall_s, 2), "wall_tok_s": round(len(got) / wall_s * 1e3, 2),
                                      "wall_ms_per_token_over_plain": round(wall_s / wall, 3),
                                      "d2h_bytes_per_round": (k + 1) * d2h_per_pos}), flush=True)
        for k in (1, 3):
            run = [first] + want[:k]
            ms = []
            for _ in range(5):
                l2b.fork(m, [own], p)
                l2b.verify_sample_ragged([own], [run], [p], [T], [TOP_P])
                ms.append(own.last_timing()[0])
            if show:
                med = float(np.median(ms))
                print(json.dumps({"what": "verify_round", "repeat": r, "k": k, "positions": k + 1,
                                  "median_device_ms": round(med, 3), "over_plain_step": round(med / base, 3),
                                  "d2h_bytes": (k + 1) * d2h_per_pos}), flush=True)
    for s in (own, ref, small, m):
        s.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
