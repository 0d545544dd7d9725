"""q8 against bf16 and fp32 device weights on the llama2-7B synthetic shape (seed 7), in one process.

The three contexts are generated on the device (26.4 GB fp32 + 13.2 GB bf16 + 7.0 GB q8) and timed
alternately, --rounds rounds:
  - decode: l2b_generate_argmax over --gen positions from an empty cache (tok/s, host clock around the call,
    which ends in a device synchronise);
  - prefill: l2b_prefill of a 256-token prompt (tok/s from l2b_last_timing's device time);
  - batch: l2b_forward_argmax_batch of 4 sessions over --batch-steps steps (tok/s over all sessions; the
    sessions of a format exist only while it is timed, so the three formats' KV caches fit beside them);
  - the dominant GEMV's bytes / time from l2b_profile_step (TB/s; the bytes are the stored ones: 4 per fp32
    weight, 2 per bf16 weight and 1 per q8 code plus 4 per scale, row padding included).
Then:
  - quantization cost: the q8 context against the fp32 context of the same (unquantized) payload: max
    relative logit difference over a 64-step teacher-forced run, and how many of 64 free-running greedy
    tokens agree;
  - parity: the q8 logits (device-generated, and uploaded from the host payload) equal, bit for bit, those
    of an fp32 context of the host payload with its matrices dequantized (l2b_round_q8_host), at 4
    positions; the q8 upload's l2b_load_stats.
Card name, power limit and max SM clock are read in the same run.  Prints one JSON line per measurement.
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
import llama2_zig_b200 as l2b  # noqa: E402
from llama2_zig_b200.checkpoint import shape_checkpoint  # noqa: E402

SEED = 7


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def decode(t, n):
    t.reset()
    t0 = time.perf_counter()
    out = t.generate_argmax(1, 0, n, stop_on_bos=False)
    return len(out) / (time.perf_counter() - t0)


def prefill(t, toks):
    t.reset()
    t.prefill(toks, want_logits=False)
    ms, _ = t.last_timing()
    return len(toks) / (ms / 1e3)


def batch(sessions, n):
    toks = [1] * len(sessions)
    for s in sessions:
        s.reset()
    t0 = time.perf_counter()
    for pos in range(n):
        toks = l2b.forward_argmax_batch(sessions, toks, [pos] * len(sessions))
    return n * len(sessions) / (time.perf_counter() - t0)


def gemv_tbs(t):
    t.reset()
    prof = t.profile_step(1, 0)
    total = {}
    for name, _, ms, by in prof:                              # the GEMV that streams the most bytes per step
        m, b = total.get(name, (0.0, 0))
        total[name] = (m + ms, b + by)
    name = max(total, key=lambda k: total[k][1])
    ms, by = total[name]
    return name, by / (ms / 1e3) / 1e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gen", type=int, default=128)
    ap.add_argument("--batch-steps", type=int, default=32)
    a = ap.parse_args()
    ck = shape_checkpoint("llama2-7B")
    gpu = card()
    print(json.dumps({"card": gpu}), flush=True)
    ctx = {k: l2b.Transformer(ck, synthetic_seed=SEED, weight_format=k) for k in ("f32", "bf16", "q8")}
    for k, t in ctx.items():
        ms, nb = t.load_stats()
        fmt, n_rounded = t.weight_info()
        print(json.dumps({"format": k, "create_ms": ms, "n_rounded": n_rounded, "step_weight_bytes": t.step_bytes(0)[0]}),
              flush=True)
    prompt = [(i * 7919) % 31999 + 1 for i in range(256)]
    res = {k: {"decode": [], "prefill": [], "batch4": [], "gemv_tbs": []} for k in ctx}
    for k, t in ctx.items():                                  # warm-up of every shape
        decode(t, 8); prefill(t, prompt[:8])
    for r in range(a.rounds):
        for k, t in ctx.items():
            res[k]["decode"].append(decode(t, a.gen))
            res[k]["prefill"].append(prefill(t, prompt))
            sess = [t.session() for _ in range(4)]
            batch(sess, 2)                                    # warm-up
            res[k]["batch4"].append(batch(sess, a.batch_steps))
            for s in sess:
                s.close()
            name, tbs = gemv_tbs(t)
            res[k]["gemv_tbs"].append(tbs)
            res[k]["gemv"] = name
    for k in ctx:
        print(json.dumps({"format": k, "card": gpu, **{m: (v if isinstance(v, str) else [round(x, 3) for x in v])
                                                      for m, v in res[k].items()}}), flush=True)
    ctx["bf16"].close()

    # quantization cost: q8 against the fp32 context of the same payload
    b, f = ctx["q8"], ctx["f32"]
    b.reset(); f.reset()
    toks = [1] + prompt[:63]
    worst = 0.0
    for pos, tok in enumerate(toks):
        lb, lf = b.forward(tok, pos), f.forward(tok, pos)
        worst = max(worst, float(np.max(np.abs(lb - lf)) / np.max(np.abs(lf))))
    gb, gf = decode_tokens(b), decode_tokens(f)
    print(json.dumps({"quantization_cost": {"max_rel_logit_diff": worst, "greedy_agree": int((gb == gf).sum()),
                                        "greedy_steps": 64,
                                        "first_disagreement": int(np.argmax(gb != gf)) if (gb != gf).any() else None}}),
          flush=True)
    f.close()

    # parity: the q8 context against an fp32 context of the dequantized host payload
    data = l2b.synth_checkpoint_host(ck, SEED)
    n_changed = 0
    for off, rows, cols in matrix_shapes(ck):
        n_changed += l2b.round_q8_host(data[off:off + rows * cols].reshape(rows, cols))
    ck.data = data
    same = True
    with l2b.Transformer(ck) as r:
        b.reset()
        for pos, tok in enumerate(toks[:4]):
            same &= np.array_equal(b.forward(tok, pos).view(np.uint32), r.forward(tok, pos).view(np.uint32))
        # the q8 upload path: quantization in the pinned stage fill (l2b_load_stats); the dequantized payload
        # quantizes to itself, so it changes no weight
        with l2b.Transformer(ck, weight_format="q8") as u:
            ms, nb = u.load_stats()
            print(json.dumps({"q8_upload": {"ms": ms, "bytes": nb, "n_changed": u.weight_info()[1],
                                            "device_n_changed": b.weight_info()[1], "host_n_changed": n_changed}}),
                  flush=True)
            u.reset(); r.reset()
            for pos, tok in enumerate(toks[:4]):
                same &= np.array_equal(u.forward(tok, pos).view(np.uint32), r.forward(tok, pos).view(np.uint32))
        ck.data = None
    print(json.dumps({"parity_bitwise_4_positions": bool(same)}), flush=True)
    b.close()


def decode_tokens(t):
    t.reset()
    return t.generate_argmax(1, 0, 64, stop_on_bos=False)


def matrix_shapes(ck):
    """(offset, rows, cols) of each matrix tensor of a payload (a stacked [L][rows][cols] tensor is L * rows rows)."""
    d, h, L, V = ck.dim, ck.hidden_dim, ck.n_layers, ck.vocab_size
    kvd = d // ck.n_heads * ck.n_kv_heads
    parts = [(V, d), ("g", L * d), (L * d, d), (L * kvd, d), (L * kvd, d), (L * d, d), ("g", L * d),
             (L * h, d), (L * d, h), (L * h, d), ("g", d), ("g", ck.seq_len * (d // ck.n_heads))]
    if not ck.shared_weights:
        parts.append((V, d))
    off = 0
    for rows, n in parts:
        if rows == "g":
            off += n
        else:
            yield off, rows, n
            off += rows * n


if __name__ == "__main__":
    main()
