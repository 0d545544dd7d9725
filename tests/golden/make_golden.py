"""Regenerates the committed golden fixtures from the CPU oracle (NOT from the Zig binary:
no Zig toolchain exists for this project, see oracle/llama2_oracle.h "Pinning status").

The checkpoint is the stories15M-shaped synthetic one of oracle_lib.write_stories15m_checkpoint
(seed oracle_lib.STORIES15M_SEED), so the fixtures and the tests need no file from outside the tree.

  stories15M_t0_tokens.json  token stream of `llama2 <checkpoint> -t 0` (no prompt) as the
                             oracle produces it; identical for W in {4,8,16}, strict/optimized
                             float mode.  `terminator` is 1 when BOS ended the stream, else null.
  stories15M_logits.npz      logits of selected positions along that stream (every 16th logit
                             + the top-32), oracle strict W=8.

  python tests/golden/make_golden.py
"""
import hashlib
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_lib as O  # noqa: E402

POSITIONS = [0, 1, 2, 50, 98, 150, 220, 221]


def main():
    O.build_oracle()
    with tempfile.TemporaryDirectory() as tmp:
        write(O.write_stories15m_checkpoint(os.path.join(tmp, "stories15M.bin")))


def write(ckpt):
    streams = {}
    for kind in ("strict", "fast"):
        cfg, shared, data = O.read_checkpoint(ckpt, kind)
        for W in (4, 8, 16):
            m = O.OracleModel(cfg, data, shared, W=W, kind=kind)
            calls, out, _ = m.generate(1, 256)
            streams[(kind, W)] = (calls, out[:calls].tolist())
            m.close()
    ref = streams[("strict", 8)]
    assert all(v == ref for v in streams.values()), "variants disagree"
    calls, nexts = ref
    terminator = 1 if nexts[-1] == 1 else None
    toks = np.array(nexts[:-1] if terminator else nexts, dtype="<u4")
    sha = hashlib.sha256(toks.tobytes()).hexdigest()
    with open(os.path.join(HERE, "stories15M_t0_tokens.json"), "w") as f:
        json.dump({"checkpoint": f"stories15M shape, synthetic weights, seed {O.STORIES15M_SEED}",
                   "checkpoint_bytes": os.path.getsize(ckpt),
                   "prompt": None, "temperature": 0, "first_token": 1, "forward_calls": calls,
                   "tokens": toks.tolist(), "terminator": terminator, "sha256_le_u32": sha,
                   "produced_by": "oracle strict W=8 (== W 4/16, == optimized float mode)"}, f, indent=1)
    print("tokens", len(toks), sha)

    cfg, shared, data = O.read_checkpoint(ckpt, "strict")
    m = O.OracleModel(cfg, data, shared, W=8, kind="strict")
    token, keep = 1, {}
    for pos in range(max(POSITIONS) + 1):
        lg = m.forward(token, pos)
        if pos in POSITIONS:
            top = np.argsort(-lg, kind="stable")[:32].astype(np.int32)
            keep[f"p{pos}_strided"] = lg[::16].copy()
            keep[f"p{pos}_top_idx"] = top
            keep[f"p{pos}_top_val"] = lg[top].copy()
        token = nexts[pos]
    np.savez_compressed(os.path.join(HERE, "stories15M_logits.npz"), positions=np.array(POSITIONS), **keep)
    print("logits fixture written")


if __name__ == "__main__":
    main()
