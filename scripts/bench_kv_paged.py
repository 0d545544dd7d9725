"""Paged against contiguous KV caches on the llama2-7B synthetic shape (seed 7, bf16 weights), in one process.

For fp32 and bf16 KV, a contiguous and a paged context of the same synthetic weights are created and measured
alternately, --rounds rounds:
  - decode: l2b_prefill fills the cache to T0, then l2b_generate_argmax runs --gen positions (tok/s, host clock
    around the call, which ends in a device synchronise), at T0 = 128, 1024, 2016 (seq_len 2048) and 4000
    (seq_len 4096), with the attention kernels' device time per layer from l2b_profile_step;
  - fork: l2b_fork of n_pos in {256, 1024, 2048} (capped at seq_len) to 1, 3 and 7 destinations, the device
    time l2b_last_timing reports (a paged fork copies at most 63 rows per destination);
  - batch: l2b_forward_argmax_batch of 4 sessions forked at T0 = 2000, --batch-steps steps (tok/s over all);
  - memory of best-of-8 (a 1984-token prompt, 64 new tokens per sample) from l2b_kv_pool_info, against
    nine contiguous caches: counted, not timed.
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
LAYOUTS = ("contiguous", "paged")


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


def attention_ms(t, toks, t0):
    prof = t.profile_step(toks[t0], t0)
    ms = [m for name, _, m, _ in prof if name in ("attention", "attn_wo")]
    return sum(ms) / len(ms)


def fork_ms(t, toks, n_pos, n_dst):
    t.reset()
    t.prefill(toks[:n_pos], 0, want_logits=False)
    dst = [t.session() for _ in range(n_dst)]
    try:
        l2b.fork(t, dst, n_pos)                                # warm-up
        l2b.fork(t, dst, n_pos)
        return t.last_timing()[0]
    finally:
        for d in dst:
            d.close()


def batch(t, toks, t0, n):
    sess = [t.session() for _ in range(4)]
    try:
        sess[0].prefill(toks[:t0], 0, want_logits=False)
        l2b.fork(sess[0], sess[1:], t0)
        nxt = [toks[t0]] * 4
        l2b.forward_argmax_batch(sess, nxt, [t0] * 4)
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
            contiguous = 9 * 2 * ck.n_layers * ck.seq_len * ck.dim * (2 if kv == "bf16" else 4)
            return {"kv": kv, "pages_in_use": info["pages_in_use"], "page_bytes": info["page_bytes"],
                    "paged_GiB": info["pages_in_use"] * info["page_bytes"] / 2**30, "contiguous_GiB": contiguous / 2**30}
        finally:
            for d in dst:
                d.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--gen", type=int, default=32)
    ap.add_argument("--batch-steps", type=int, default=16)
    ap.add_argument("--kv", default="f32,bf16")
    ap.add_argument("--seq-lens", default="2048,4096")
    a = ap.parse_args()
    gpu = card()
    print(json.dumps({"card": gpu}), flush=True)
    base = shape_checkpoint("llama2-7B")
    for S in [int(x) for x in a.seq_lens.split(",")]:
        ck = shape_checkpoint((base.dim, base.hidden_dim, base.n_layers, base.n_heads, base.n_kv_heads,
                               base.vocab_size if base.shared_weights else -base.vocab_size, S))
        toks = stream(S, ck.vocab_size)
        points = [128, 1024, 2016] if S == 2048 else [4000]
        for kv in a.kv.split(","):
            ctx = {lay: l2b.Transformer(ck, synthetic_seed=SEED, weight_format="bf16", kv_format=kv, kv_layout=lay)
                   for lay in LAYOUTS}
            for t in ctx.values():
                decode(t, toks, 0, 4)                          # warm-up
            res = {lay: {"decode": {p: [] for p in points}, "attn_ms": {p: [] for p in points}, "batch4": [],
                         "fork_ms": {}} for lay in LAYOUTS}
            for _ in range(a.rounds):
                for p in points:
                    for lay, t in ctx.items():
                        res[lay]["decode"][p].append(decode(t, toks, p, a.gen))
                        res[lay]["attn_ms"][p].append(attention_ms(t, toks, p + a.gen - 1))
                if S == 2048:
                    for lay, t in ctx.items():
                        res[lay]["batch4"].append(batch(t, toks, 2000, a.batch_steps))
            if S == 2048:
                for n_pos in (256, 1024, 2048):
                    for nd in (1, 3, 7):
                        for lay, t in ctx.items():
                            res[lay]["fork_ms"][f"{n_pos}x{nd}"] = round(fork_ms(t, toks, min(n_pos, S), nd), 4)
            for lay in LAYOUTS:
                r = res[lay]
                print(json.dumps({"seq_len": S, "weights": "bf16", "kv": kv, "layout": lay, "card": gpu,
                                  "decode_tok_s": {p: [round(x, 2) for x in v] for p, v in r["decode"].items()},
                                  "attn_ms_per_layer": {p: [round(x, 4) for x in v] for p, v in r["attn_ms"].items()},
                                  "batch4_tok_s": [round(x, 2) for x in r["batch4"]], "fork_ms": r["fork_ms"]}),
                      flush=True)
            for t in ctx.values():
                t.close()
            if S == 2048:
                print(json.dumps({"best_of_8": best_of_8(ck, kv, toks), "card": gpu}), flush=True)


if __name__ == "__main__":
    np.seterr(all="ignore")
    main()
