"""e4m3 against bf16 KV caches on the llama2-7B synthetic shape (seed 7), in one process.

For seq_len 2048 and 4096 and for each --weights format, a bf16-KV and an e4m3-KV context (unit scales) of the
same synthetic weights are created and measured alternately, --rounds rounds:
  - decode: l2b_prefill fills the cache to T0, then l2b_generate_argmax runs --gen positions from there (tok/s,
    host clock around the call, which ends in a device synchronise), at T0 = 128, 1024, 2016 (seq_len 2048) and
    4000 (seq_len 4096);
  - attention per layer: the "attention" / "attn_wo" kernels' device time from l2b_profile_step at the last
    decoded position (us per layer, and the bytes l2b_profile_step counts over that time);
  - batch: l2b_forward_argmax_batch of 4 sessions forked at T0 = 2000, --batch-steps steps (tok/s over all);
  - the cache bytes of one context (l2b_kv_info).
Then, at seq_len 2048 (counted, not timed): the pages and bytes a paged best-of-8 from a 1984-token prompt holds
(l2b_kv_pool_info) in bf16 and e4m3.  And, with bf16 weights, the accuracy cost against an fp32-KV context of the
same payload: the max relative logit difference over a teacher-forced run of the whole context and how many of 64
free-running greedy tokens agree, for bf16 KV, e4m3 KV with unit scales and e4m3 KV with calibrated scales.  The
calibrated scales are each layer's amax / 448 of the fp32-KV context's K and V after a calibration prompt (a
token stream other than the evaluated one), computed here and not in the library.
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
KVS = ("bf16", "e4m3")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def stream(n, V, mul=7919):
    return [1] + [(i * mul) % (V - 1) + 1 for i in range(1, n)]


def decode(t, toks, t0, n):
    t.reset()
    if t0 > 0:
        t.prefill(toks[:t0], 0, want_logits=False)
    start = time.perf_counter()
    out = t.generate_argmax(toks[t0], t0, n, stop_on_bos=False)
    return len(out) / (time.perf_counter() - start)


def attention(t, toks, t0):
    """(us per layer, GB/s counted by l2b_profile_step) of the attention kernels of one step at position t0."""
    prof = t.profile_step(toks[t0], t0)
    rows = [(ms, by) for name, _, ms, by in prof if name in ("attention", "attn_wo")]
    ms = sum(r[0] for r in rows)
    return 1e3 * ms / len(rows), sum(r[1] for r in rows) / (ms / 1e3) / 1e9


def batch(t, toks, t0, n):
    sess = [t.session() for _ in range(4)]
    try:
        sess[0].prefill(toks[:t0], 0, want_logits=False)
        l2b.fork(sess[0], sess[1:], t0)
        nxt = [toks[t0]] * 4
        l2b.forward_argmax_batch(sess, nxt, [t0] * 4)          # warm-up
        start = time.perf_counter()
        for k in range(n):
            nxt = l2b.forward_argmax_batch(sess, nxt, [t0 + 1 + k] * 4)
        return 4 * n / (time.perf_counter() - start)
    finally:
        for s in sess:
            s.close()


def best_of_8(ck, kv, toks):
    with l2b.Transformer(ck, synthetic_seed=SEED, weight_format="bf16", kv_format=kv, kv_layout="paged") as m:
        m.prefill(toks[:1984], 0, want_logits=False)
        dst = [m.session() for _ in range(8)]
        try:
            l2b.fork(m, dst, 1983)
            l2b.generate_argmax_batch(dst, [toks[1983]] * 8, [1983] * 8, 64, stop_on_bos=False)
            info = m.kv_pool_info()
            return {"kv": kv, "pages_in_use": info["pages_in_use"], "page_bytes": info["page_bytes"],
                    "paged_GiB": info["pages_in_use"] * info["page_bytes"] / 2**30}
        finally:
            for d in dst:
                d.close()


def calibrated_scales(f, ck, toks):
    """per layer amax / 448 of f's (an fp32-KV context) K and V after prefilling toks"""
    f.reset()
    f.prefill(toks, 0, want_logits=False)
    n = len(toks)
    s = np.empty((ck.n_layers, 2), np.float32)
    for j, name in enumerate(("key_cache", "value_cache")):
        c = f.state(name).reshape(ck.n_layers, ck.seq_len, -1)[:, :n]
        s[:, j] = np.abs(c).max(axis=(1, 2)) / np.float32(448)
    f.reset()
    return s


def accuracy(t, f, toks):
    t.reset(); f.reset()
    worst = 0.0
    for pos, tok in enumerate(toks):
        lt, lf = t.forward(tok, pos), f.forward(tok, pos)
        worst = max(worst, float(np.max(np.abs(lt - lf)) / np.max(np.abs(lf))))
    t.reset(); f.reset()
    gt = t.generate_argmax(1, 0, 64, stop_on_bos=False)
    gf = f.generate_argmax(1, 0, 64, stop_on_bos=False)
    t.reset(); f.reset()
    return {"max_rel_logit_diff": worst, "teacher_forced_positions": len(toks),
            "greedy_agree": int((gt == gf).sum()), "greedy_steps": 64,
            "first_disagreement": int(np.argmax(gt != gf)) if (gt != gf).any() else None}


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
        points = [128, 1024, 2016] if S == 2048 else [4000]
        for wf in a.weights.split(","):
            ctx = {kv: l2b.Transformer(ck, synthetic_seed=SEED, weight_format=wf, kv_format=kv) for kv in KVS}
            for kv, t in ctx.items():
                print(json.dumps({"seq_len": S, "weights": wf, "kv": kv, "cache_bytes": t.kv_info()[1],
                                  "step_kv_bytes_at_2047": t.step_bytes(min(2047, S - 1))[1]}), flush=True)
                decode(t, toks, 0, 4)                         # warm-up
            res = {kv: {"decode": {p: [] for p in points}, "attn_us": {p: [] for p in points},
                        "attn_gbs": {p: [] for p in points}, "batch4": []} for kv in ctx}
            for _ in range(a.rounds):
                for p in points:
                    for kv, t in ctx.items():
                        res[kv]["decode"][p].append(decode(t, toks, p, a.gen))
                        us, gbs = attention(t, toks, p + a.gen - 1)
                        res[kv]["attn_us"][p].append(us)
                        res[kv]["attn_gbs"][p].append(gbs)
                if S == 2048:
                    for kv, t in ctx.items():
                        res[kv]["batch4"].append(batch(t, toks, 2000, a.batch_steps))
            for kv in ctx:
                r = res[kv]
                print(json.dumps({"seq_len": S, "weights": wf, "kv": kv, "card": gpu,
                                  "decode_tok_s": {p: [round(x, 2) for x in v] for p, v in r["decode"].items()},
                                  "attn_us_per_layer": {p: [round(x, 2) for x in v] for p, v in r["attn_us"].items()},
                                  "attn_GB_s": {p: [round(x, 1) for x in v] for p, v in r["attn_gbs"].items()},
                                  "batch4_tok_s": [round(x, 2) for x in r["batch4"]]}), flush=True)
            if S == 2048 and wf == "bf16" and not a.no_accuracy:
                f = l2b.Transformer(ck, synthetic_seed=SEED, weight_format=wf)
                cal = l2b.Transformer(ck, synthetic_seed=SEED, weight_format=wf, kv_format="e4m3")
                try:
                    scales = calibrated_scales(f, ck, stream(256, ck.vocab_size, mul=104729))
                    cal.set_kv_scales(scales)
                    for what, t in (("bf16", ctx["bf16"]), ("e4m3-unit", ctx["e4m3"]), ("e4m3-calibrated", cal)):
                        print(json.dumps({"seq_len": S, "weights": wf, "kv": what, "card": gpu,
                                          "accuracy_vs_f32_kv": accuracy(t, f, toks)}), flush=True)
                    print(json.dumps({"calibrated_scales_range": [float(scales.min()), float(scales.max())]}), flush=True)
                finally:
                    f.close(); cal.close()
            for t in ctx.values():
                t.close()
        if S == 2048:
            for kv in KVS:
                print(json.dumps({"best_of_8": best_of_8(ck, kv, toks), "card": gpu}), flush=True)


if __name__ == "__main__":
    np.seterr(all="ignore")
    main()
