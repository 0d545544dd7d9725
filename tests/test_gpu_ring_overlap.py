"""GPU: the TMA-ring GEMV's shared-memory layout does not change what it computes.

gemv_tma_kernel streams weights through a ring of 4-row (16 KB) slots, two per 8-row tile and column
step, whose depth launch_gemv picks from the shared memory of one SM, split for L2B_TMA_CTAS ring
CTAs.  Every consumer thread reads the same columns of the same rows in the same order whatever the
split or the depth, so the logits, the device argmax and the KV rows must be bit for bit those of the
default context (a whole-SM ring).
"""
import numpy as np
import pytest

from test_gpu_transformer import teacher_tokens
from test_gpu_variants import l2b_env

pytestmark = pytest.mark.gpu

# TinyLlama's layer shape, 2 layers: every decode epilogue on the ring (qkv with GQA, wo and w2 with the
# residual add, w13 with SiLU, w2's 5632-float input, the odd-sized argmax classifier).  The qkv rows
# leave some CTAs a 2-row last tile, whose second slot lands no bytes.
SHAPE = (2048, 5632, 2, 32, 4, -32003, 300)
N_POS = 260                      # crosses the 256-position attention split
CONFIGS = {
    "ctas2": {"L2B_TMA_CTAS": "2"},       # ring sized for two CTAs per SM: 4 to 6 slots
    "stages3": {"L2B_TMA_STAGES": "3"},   # a column step's two slots straddle the ring's wrap
}


def run(l2b, env):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint(SHAPE)
    toks = teacher_tokens(N_POS, ck.vocab_size)
    with l2b_env(env), l2b.Transformer(ck, synthetic_seed=5) as t:
        logits = np.stack([t.forward(tok, pos) for pos, tok in enumerate(toks)])
        amax = [t.forward_argmax(tok, pos) for pos, tok in enumerate(toks)]
        return logits, amax, t.state("key_cache"), t.state("value_cache")


_default = {}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_ring_layout_is_bitwise(l2b, config):
    if "ref" not in _default:
        _default["ref"] = run(l2b, {})
    want = _default["ref"]
    got = run(l2b, CONFIGS[config])
    assert np.array_equal(got[0], want[0])
    assert got[1] == want[1] == [int(np.argmax(r)) for r in want[0]]
    assert np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3])
