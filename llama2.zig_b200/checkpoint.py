"""Legacy llama2.c checkpoint files: 28-byte header + flat fp32 payload.

Mirrors what the reference's host does before the hot path starts
(src/main.zig:936-967: read ConfigReader, sign of vocab_size => shared
classifier, slurp the rest of the file).  Host-side plumbing only; no arithmetic.
"""
import os
from dataclasses import dataclass

import numpy as np

# (dim, hidden_dim, n_layers, n_heads, n_kv_heads, vocab_size(header sign!), seq_len); SURVEY.md 8
MODEL_SHAPES = {
    "stories15M": (288, 768, 6, 6, 6, 32000, 256),
    "stories110M": (768, 2048, 12, 12, 12, 32000, 1024),
    "llama2-7B": (4096, 11008, 32, 32, 32, -32000, 2048),
}


@dataclass
class Checkpoint:
    dim: int
    hidden_dim: int
    n_layers: int
    n_heads: int
    n_kv_heads: int
    vocab_size: int
    seq_len: int
    shared_weights: bool
    data: np.ndarray  # float32 payload after the header (may be a memmap), or None

    @property
    def shape_tuple(self):
        return (self.dim, self.hidden_dim, self.n_layers, self.n_heads, self.n_kv_heads,
                self.vocab_size, self.seq_len)


def shape_checkpoint(name_or_tuple, data=None):
    t = MODEL_SHAPES[name_or_tuple] if isinstance(name_or_tuple, str) else tuple(name_or_tuple)
    dim, hid, L, H, KV, V, S = t
    return Checkpoint(dim, hid, L, H, KV, abs(V), S, V > 0, data)


def read_checkpoint(path, mmap=True):
    """Header parse of src/main.zig:937-946; payload as float32 (memory-mapped by default)."""
    with open(path, "rb") as f:
        hdr = np.frombuffer(f.read(28), dtype="<i4")
    if hdr.size != 7:
        raise ValueError(f"{path}: shorter than the 28-byte header")
    dim, hid, L, H, KV, V, S = (int(v) for v in hdr)
    shared = V > 0                       # :943
    V = abs(V)                           # :944
    n = (os.path.getsize(path) - 28) // 4
    if mmap:
        data = np.memmap(path, dtype="<f4", mode="r", offset=28, shape=(n,))
    else:
        data = np.fromfile(path, dtype="<f4", offset=28, count=n)
    return Checkpoint(dim, hid, L, H, KV, V, S, shared, data)
