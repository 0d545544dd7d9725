"""bf16 against fp32 KV caches on the llama2-7B synthetic shape (seed 7), in one process.

For seq_len 2048 and 4096 and for bf16 and q8 weights, an fp32-KV and a bf16-KV context of the same
synthetic weights are created and measured alternately, --rounds rounds:
  - decode: l2b_prefill fills the cache to T0, then l2b_generate_argmax runs --gen positions from there (tok/s,
    host clock around the call, which ends in a device synchronise), at T0 = 128, 1024, 2048 and, at seq_len
    4096, 4000 (each capped at seq_len - gen);
  - attention per layer: the "attention" kernels' device time and bytes from l2b_profile_step at T0 (ms per
    layer, and bytes / time: 4 or 2 bytes per cache element read);
  - batch: l2b_forward_argmax_batch of 4 sessions at T0 = 2000 (one prefill, then l2b_fork to the others),
    --batch-steps steps (tok/s over all sessions);
  - the cache bytes of one context (l2b_kv_info).
Then, at seq_len 2048, the accuracy cost: the bf16-KV context against the fp32-KV context of the same payload
and weight format, the max relative logit difference over a teacher-forced run to the end of the context,
and how many of 64 free-running greedy tokens agree.
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


def stream(n, V):
    return [1] + [(i * 7919) % (V - 1) + 1 for i in range(1, n)]


def decode(t, toks, t0, n):
    t.reset()
    if t0 > 0:
        t.prefill(toks[:t0], 0, want_logits=False)
    start = time.perf_counter()
    out = t.generate_argmax(toks[t0], t0, n, stop_on_bos=False)
    return len(out) / (time.perf_counter() - start)


def attention(t, toks, t0):
    """(ms per layer, GB/s) of the attention kernels of one step at position t0."""
    prof = t.profile_step(toks[t0], t0)
    rows = [(ms, by) for name, _, ms, by in prof if name in ("attention", "attn_wo")]
    ms = sum(r[0] for r in rows)
    by = sum(r[1] for r in rows)
    return ms / len(rows), by / (ms / 1e3) / 1e9


def batch(t, toks, t0, n):
    sess = [t.session() for _ in range(4)]
    try:
        sess[0].prefill(toks[:t0], 0, want_logits=False)
        l2b.fork(sess[0], sess[1:], t0)
        nxt = [toks[t0]] * 4
        l2b.forward_argmax_batch(sess, nxt, [t0] * 4)          # warm-up
        start = time.perf_counter()
        for k in range(n):
            nxt = l2b.forward_argmax_batch(sess, nxt, [t0 + k] * 4)
        return 4 * n / (time.perf_counter() - start)
    finally:
        for s in sess:
            s.close()


def accuracy(b, f, toks):
    b.reset(); f.reset()
    worst = 0.0
    for pos, tok in enumerate(toks):
        lb, lf = b.forward(tok, pos), f.forward(tok, pos)
        worst = max(worst, float(np.max(np.abs(lb - lf)) / np.max(np.abs(lf))))
    b.reset(); f.reset()
    gb = b.generate_argmax(1, 0, 64, stop_on_bos=False)
    gf = f.generate_argmax(1, 0, 64, stop_on_bos=False)
    return {"max_rel_logit_diff": worst, "teacher_forced_positions": len(toks),
            "greedy_agree": int((gb == gf).sum()), "greedy_steps": 64,
            "first_disagreement": int(np.argmax(gb != gf)) if (gb != gf).any() else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--gen", type=int, default=32)
    ap.add_argument("--batch-steps", type=int, default=16)
    ap.add_argument("--seq-lens", default="2048,4096")
    ap.add_argument("--weights", default="bf16,q8")
    ap.add_argument("--no-accuracy", action="store_true")
    a = ap.parse_args()
    gpu = card()
    print(json.dumps({"card": gpu}), flush=True)
    base = shape_checkpoint("llama2-7B")
    for S in [int(x) for x in a.seq_lens.split(",")]:
        ck = shape_checkpoint((base.dim, base.hidden_dim, base.n_layers, base.n_heads, base.n_kv_heads,
                               base.vocab_size if base.shared_weights else -base.vocab_size, S))
        toks = stream(S, ck.vocab_size)
        points = [p for p in (128, 1024, 2048) if p <= S] + ([4000] if S >= 4096 else [])
        points = [min(p, S - a.gen) for p in points]
        for wf in a.weights.split(","):
            ctx = {kv: l2b.Transformer(ck, synthetic_seed=SEED, weight_format=wf, kv_format=kv) for kv in ("f32", "bf16")}
            for kv, t in ctx.items():
                print(json.dumps({"seq_len": S, "weights": wf, "kv": kv, "cache_bytes": t.kv_info()[1],
                                  "step_kv_bytes_at_2047": t.step_bytes(min(2047, S - 1))[1]}), flush=True)
                decode(t, toks, 0, 4)                         # warm-up
            res = {kv: {"decode": {p: [] for p in points}, "attn_ms": {p: [] for p in points},
                        "attn_gbs": {p: [] for p in points}, "batch4": []} for kv in ctx}
            for _ in range(a.rounds):
                for p in points:
                    for kv, t in ctx.items():
                        res[kv]["decode"][p].append(decode(t, toks, p, a.gen))
                        ms, gbs = attention(t, toks, p + a.gen - 1)
                        res[kv]["attn_ms"][p].append(ms)
                        res[kv]["attn_gbs"][p].append(gbs)
                for kv, t in ctx.items():
                    res[kv]["batch4"].append(batch(t, toks, min(2000, S - a.batch_steps - 2), a.batch_steps))
            for kv in ctx:
                r = res[kv]
                print(json.dumps({"seq_len": S, "weights": wf, "kv": kv, "card": gpu,
                                  "decode_tok_s": {p: [round(x, 2) for x in v] for p, v in r["decode"].items()},
                                  "attn_ms_per_layer": {p: [round(x, 4) for x in v] for p, v in r["attn_ms"].items()},
                                  "attn_GB_s": {p: [round(x, 1) for x in v] for p, v in r["attn_gbs"].items()},
                                  "batch4_tok_s": [round(x, 2) for x in r["batch4"]]}), flush=True)
            if S == 2048 and not a.no_accuracy:
                print(json.dumps({"seq_len": S, "weights": wf,
                                  "accuracy": accuracy(ctx["bf16"], ctx["f32"], toks)}), flush=True)
            for t in ctx.values():
                t.close()


if __name__ == "__main__":
    main()
