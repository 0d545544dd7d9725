"""Tensor-parallel shard plan of the decode step (SURVEY.md 8e) — the host-side description of
what `materialize()` in csrc/llama2_b200.cu uploads for one rank.  Pure Python, no arithmetic of
the hot path: used by the CPU (gloo) tests of the N>1 logic and for byte accounting.

Column-parallel (split output rows): wq, wk, wv by heads; w1, w3 by hidden; wcls by vocab.
Row-parallel (split input columns): wo (input = local heads), w2 (input = local hidden).
Replicated: token_embedding_table, rms_att, rms_ffn, rms_final.
All-reduce (sum over ranks, `dim` floats): after wo and after w2 — two per layer.
"""
from dataclasses import dataclass


@dataclass(frozen=True)
class Slice2D:
    row0: int
    row1: int
    col0: int
    col1: int

    @property
    def shape(self):
        return (self.row1 - self.row0, self.col1 - self.col0)


def validate(ck, world):
    hs = ck.dim // ck.n_heads
    if world not in (1, 2, 4, 8):
        raise ValueError("world_size must be 1, 2, 4 or 8")
    if ck.n_kv_heads % world or ck.hidden_dim % world or (ck.hidden_dim // world) % 4 or ck.vocab_size % world:
        raise ValueError("shape does not divide over world_size")
    return hs


def shard_plan(ck, rank, world):
    """Per-layer 2-D windows (rows, cols) of each tensor that `rank` holds."""
    hs = validate(ck, world)
    dim, hid, V = ck.dim, ck.hidden_dim, ck.vocab_size
    kvd = hs * ck.n_kv_heads
    q_loc, kv_loc, hid_loc, v_loc = dim // world, kvd // world, hid // world, V // world
    return {
        "token_embedding_table": Slice2D(0, V, 0, dim),
        "rms_att_weight": Slice2D(0, 1, 0, dim),
        "wq": Slice2D(rank * q_loc, (rank + 1) * q_loc, 0, dim),
        "wk": Slice2D(rank * kv_loc, (rank + 1) * kv_loc, 0, dim),
        "wv": Slice2D(rank * kv_loc, (rank + 1) * kv_loc, 0, dim),
        "wo": Slice2D(0, dim, rank * q_loc, (rank + 1) * q_loc),
        "rms_ffn_weight": Slice2D(0, 1, 0, dim),
        "w1": Slice2D(rank * hid_loc, (rank + 1) * hid_loc, 0, dim),
        "w2": Slice2D(0, dim, rank * hid_loc, (rank + 1) * hid_loc),
        "w3": Slice2D(rank * hid_loc, (rank + 1) * hid_loc, 0, dim),
        "rms_final_weight": Slice2D(0, 1, 0, dim),
        "wcls": Slice2D(rank * v_loc, (rank + 1) * v_loc, 0, dim),
    }


def payload_views(ck):
    """Full tensors as numpy views over the checkpoint payload, in file order
    (src/main.zig:85-112)."""
    import numpy as np
    dim, hid, L, V, S = ck.dim, ck.hidden_dim, ck.n_layers, ck.vocab_size, ck.seq_len
    hs = dim // ck.n_heads
    kvd = hs * ck.n_kv_heads
    d = ck.data
    off = 0

    def take(n, shape):
        nonlocal off
        v = np.asarray(d[off:off + n]).reshape(shape)
        off += n
        return v

    t = {}
    t["token_embedding_table"] = take(V * dim, (V, dim))
    t["rms_att_weight"] = take(L * dim, (L, dim))
    t["wq"] = take(L * dim * dim, (L, dim, dim))
    t["wk"] = take(L * kvd * dim, (L, kvd, dim))
    t["wv"] = take(L * kvd * dim, (L, kvd, dim))
    t["wo"] = take(L * dim * dim, (L, dim, dim))
    t["rms_ffn_weight"] = take(L * dim, (L, dim))
    t["w1"] = take(L * hid * dim, (L, hid, dim))
    t["w2"] = take(L * dim * hid, (L, dim, hid))
    t["w3"] = take(L * hid * dim, (L, hid, dim))
    t["rms_final_weight"] = take(dim, (dim,))
    off += 2 * (S * hs // 2)
    t["wcls"] = t["token_embedding_table"] if ck.shared_weights else take(V * dim, (V, dim))
    return t


def weight_bytes_per_token(ck, world=1):
    """Algorithmic weight bytes one rank streams per token (SURVEY.md 8d formula, sharded)."""
    hs = validate(ck, world)
    dim, hid, L, V = ck.dim, ck.hidden_dim, ck.n_layers, ck.vocab_size
    kvd = hs * ck.n_kv_heads
    per_layer = (dim // world) * dim + 2 * (kvd // world) * dim + dim * (dim // world) + 3 * (hid // world) * dim + 2 * dim
    return 4 * (L * per_layer + dim + (V // world) * dim)
