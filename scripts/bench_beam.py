"""Beam search on the llama2-7B synthetic shape (seed 7, bf16 weights, bf16 paged KV, seq_len 2048), in one process.

For prompts of 256 and 1984 tokens and B in {1, 2, 4, 8} beams, --steps steps (stop_on_bos 0), alternately,
--rounds rounds:
  - beam: l2b_beam_search from the prompt; its device time per step (l2b_last_timing spans the whole call, the
    host work between steps included) and the host clock around the call;
  - batch: l2b_generate_argmax_batch of B forks of the same prompt over the same steps: the same weight passes
    (B vectors, 4 per pass) without the selection and the page remap, so the difference to beam is the
    search's overhead (top-k kernel, one host round trip per step, page-table uploads, page copies).
Then one beam search per point under torch.profiler (CUDA activities): the device time per step of the page
copies (kv_fork_kernel: the copy-on-write of kv_reserve) and of logprob_topk_batch_kernel, on their own.
The pages held at the end (l2b_kv_pool_info) are set against B contiguous caches.  Card name, power limit and
max SM clock are read in the same run.  Prints one JSON line per point.
"""
import argparse
import json
import os
import subprocess
import sys
import time

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


def beam(m, beams, tok, pos, steps):
    start = time.perf_counter()
    _, _, ran = l2b.beam_search(m, tok, pos, beams, steps, stop_on_bos=False)
    wall = time.perf_counter() - start
    return m.last_timing()[0] / ran, wall * 1e3 / ran


def batch(m, forks, tok, pos, steps):
    l2b.fork(m, forks, pos)
    start = time.perf_counter()
    l2b.generate_argmax_batch(forks, [tok] * len(forks), [pos] * len(forks), steps, stop_on_bos=False)
    wall = time.perf_counter() - start
    return forks[0].last_timing()[0] / steps, wall * 1e3 / steps


def profiled(m, beams, tok, pos, steps):
    """device ms per step of the page copies and of the top-k kernel, and the copies per step"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _, _, ran = l2b.beam_search(m, tok, pos, beams, steps, stop_on_bos=False)
        torch.cuda.synchronize()
    copy_us = topk_us = 0.0
    copies = 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if "kv_fork_kernel" in e.name:
            copy_us += e.device_time
            copies += 1
        elif "logprob_topk_batch_kernel" in e.name:
            topk_us += e.device_time
    return {"cow_ms_per_step": round(copy_us / 1e3 / ran, 4), "pages_copied_per_step": round(copies / ran, 2),
            "topk_ms_per_step": round(topk_us / 1e3 / ran, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--prompts", default="256,1984")
    ap.add_argument("--beams", default="1,2,4,8")
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    gpu = card()
    print(json.dumps({"card": gpu}), flush=True)
    ck = shape_checkpoint("llama2-7B")
    ck.seq_len = 2048
    toks = stream(ck.seq_len, ck.vocab_size)
    kv_dim = ck.dim // ck.n_heads * ck.n_kv_heads
    contiguous_bytes = 2 * ck.n_layers * ck.seq_len * kv_dim * 2            # one bf16 cache, K and V
    with l2b.Transformer(ck, synthetic_seed=SEED, weight_format="bf16", kv_format="bf16", kv_layout="paged") as m:
        sess = [m.session() for _ in range(16)]
        try:
            for n_prompt in [int(x) for x in a.prompts.split(",")]:
                m.reset()
                m.prefill(toks[:n_prompt], 0, want_logits=False)
                tok, pos = toks[n_prompt], n_prompt
                steps = min(a.steps, ck.seq_len - pos)
                for B in [int(x) for x in a.beams.split(",")]:
                    beams, forks = sess[:B], sess[8:8 + B]
                    beam(m, beams, tok, pos, 2)                          # warm-up
                    batch(m, forks, tok, pos, 2)
                    res = {"beam_ms_per_step": [], "beam_wall_ms_per_step": [], "batch_ms_per_step": [],
                           "batch_wall_ms_per_step": []}
                    for _ in range(a.rounds):
                        d, w = beam(m, beams, tok, pos, steps)
                        res["beam_ms_per_step"].append(round(d, 4))
                        res["beam_wall_ms_per_step"].append(round(w, 4))
                        d, w = batch(m, forks, tok, pos, steps)
                        res["batch_ms_per_step"].append(round(d, 4))
                        res["batch_wall_ms_per_step"].append(round(w, 4))
                    for s in forks:
                        s.reset()
                    info = m.kv_pool_info()
                    res["overhead"] = round(min(res["beam_ms_per_step"]) / min(res["batch_ms_per_step"]) - 1, 4)
                    res["pages_in_use"] = info["pages_in_use"]
                    res["src_pages"] = m.kv_info()[1] // info["page_bytes"]
                    res["paged_MiB"] = round(info["pages_in_use"] * info["page_bytes"] / 2**20, 1)
                    res["contiguous_MiB"] = round(B * contiguous_bytes / 2**20, 1)
                    if not a.no_profile:
                        res.update(profiled(m, beams, tok, pos, steps))
                    for s in beams:
                        s.reset()
                    print(json.dumps({"prompt": n_prompt, "beams": B, "steps": steps, "weights": "bf16", "kv": "bf16 paged",
                                      "card": gpu, **res}), flush=True)
        finally:
            for s in sess:
                s.close()


if __name__ == "__main__":
    main()
