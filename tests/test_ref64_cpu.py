"""CPU: the strict oracle against an independent float64 forward pass (tests/ref64.py) on every shape
class the GPU suite runs, and on stress checkpoints whose numerics the synthetic weights never reach.

Every model-level GPU test compares the library with the strict oracle (oracle/llama2_oracle.c).  A
reading of src/main.zig that the oracle and the kernels shared would pass all of them.  ref64 is
written from main.zig alone and finds the tensors in the payload itself, so agreement here pins the
oracle's readings of the GQA / MQA head mapping (h / kv_mul, :369, :382), of RoPE rotating k only
for i < kv_dim (:343), of the unshared classifier after the two freq_cis blocks (:85-112), and of
contexts past the 256-position attention split and up to 4096 positions.

Stress checkpoints (`stress`): deterministic edits of a MODELS payload, each with a self-check on the
float64 run (`stress_check`) so that the stress cannot fade unnoticed if the edit is retuned:
  peaked   wq and wk scaled: most heads put > 0.9 of their weight on one position, and in some head
           past 256 positions the arg-max position lies in a later 256-position split whose maximum
           score exceeds the first split's by more than 20;
  sink     a constant embedding channel feeds one query dimension of every layer-0 head, and the
           matching key dimension reads the first teacher token's direction: every later position
           of every layer-0 head puts > 0.99 of its weight on position 0 while later splits fill;
  outliers a few embedding columns scaled up and their rms gains scaled down: max|x| / median|x| of
           the residual stream >= 100;
  loud     rms_final_weight scaled: logits span >= 40 and the teacher targets reach log-probabilities
           below -30.
"""
import numpy as np
import pytest

import ref64
from test_gpu_envelope import ENVELOPE
from test_gpu_transformer import teacher_tokens
from test_gpu_variants import MODELS, oracle_run, payload

# bound of e = max|oracle - ref64| / max|ref64| on logits and KV rows; measured up to ~1e-5 (KV rows
# of small-magnitude caches), fp32 rounding of a few hundred terms
ORACLE_TOL = 5e-5

STRESS_MODELS = ("S", "B", "hs28")
STRESS_KINDS = ("peaked", "sink", "outliers", "loud")

# ENVELOPE shapes a CPU runs in seconds (the multi-GB layer shapes are left to the GPU suite)
CPU_ENVELOPE = ("mqa64", "vocab1", "vocab2-seq1", "vocab3-2layers", "ctx4096-h32")


def _views(shape, data):
    return ref64.tensors(shape, data)


def _key_spike(w, shape, pos, kv_heads, score):
    """Raise the layer-0 score of the teacher token at `pos` by about `score` in the query heads of
    `kv_heads`.  Channel dim-1 of every embedding row becomes a constant that holds half of the row's
    energy, so after rmsnorm it is a near-constant positive input; query dimension j = hs-2 of those
    heads reads only that channel, and key dimension j reads the direction of the token's own
    normalised embedding (so other tokens add ~ score / |xn| * N(0, 1)).  Pair j is the slowest RoPE
    pair, which turns by < 0.1 rad over 520 positions.  Every position holding that token gets the
    raise: in a vocabulary shorter than the run, the token's repeats too."""
    dim, _, _, H, KV = shape[:5]
    hs, kv_mul, c, j = dim // H, H // KV, dim - 1, dim // H - 2
    w["token_embedding_table"][:, c] = np.float32(0.04 * np.sqrt(dim))     # the synthetic rows' sigma is 0.04
    e = w["token_embedding_table"][teacher_tokens(pos + 1, abs(shape[5]))[pos]].astype(np.float64)
    xn = e / np.sqrt(np.mean(e * e) + 1e-5) * w["rms_att_weight"][0]
    q_c = xn[c]
    xn[c] = 0.0
    gain = score * np.sqrt(hs) / (q_c * np.linalg.norm(xn))
    d = (xn / np.linalg.norm(xn)).astype(np.float32)
    for g in kv_heads:
        w["wk"][0, g * hs + j] = np.float32(gain) * d
        for h in range(g * kv_mul, (g + 1) * kv_mul):
            w["wq"][0, h * hs + j] = 0.0
            w["wq"][0, h * hs + j, c] = np.float32(1.0)


def stress(l2b, name, kind):
    """(shape, payload) of stress checkpoint `kind` built from MODELS[name]'s synthetic payload."""
    shape = MODELS[name][0]
    data = payload(l2b, name).data.copy()
    w = _views(shape, data)
    dim, _, L, H, KV = shape[:5]
    if kind == "peaked":
        w["wq"][:] *= np.float32(6.0)
        w["wk"][:] *= np.float32(6.0)
        if abs(shape[5]) >= MODELS[name][2]:
            # a peak in the second 256-position split (a token that also sits in the first split, as
            # in a short vocabulary, would not give one: there the scaled scores alone must)
            _key_spike(w, shape, 257, [0], PEAK_SPIKE)
    elif kind == "sink":
        _key_spike(w, shape, 0, range(KV), SINK_SPIKE)
    elif kind == "outliers":
        cols = np.array([3, dim // 3, dim // 2 + 1, dim - 5])
        s = np.float32(200.0)
        w["token_embedding_table"][:, cols] *= s
        w["rms_att_weight"][:, cols] /= s
        w["rms_ffn_weight"][:, cols] /= s
        w["rms_final_weight"][cols] /= s
    elif kind == "loud":
        w["rms_final_weight"][:] *= np.float32(4.0)
    else:
        raise ValueError(kind)
    return shape, data


SINK_SPIKE = 40.0                                   # score raise of position 0's key (a few units elsewhere)
PEAK_SPIKE = 160.0                                  # above the 6x-scaled scores' maxima of ~100


def stress_check(kind, shape, run, n):
    """The self-check of `kind` on ref64 run `run` of n positions; returns the measured stress."""
    H = shape[3]
    if kind == "peaked":
        peak = [float(np.max(p[h])) for l in run.probs for pos, p in run.probs[l].items() if pos >= 2
                for h in range(H)]
        frac = float(np.mean(np.array(peak) > 0.9))
        gap = 0.0                                     # a later split's max score above the first split's
        for l in run.scores:
            for pos, sc in run.scores[l].items():
                if pos < 256:
                    continue
                for h in range(H):
                    t = int(np.argmax(sc[h]))
                    if t >= 256:
                        gap = max(gap, float(sc[h, (t // 256) * 256:].max() - sc[h, :256].max()))
        assert frac > 0.5, frac
        assert gap > 20, gap
        return {"frac_peaked": frac, "split_gap": gap}
    if kind == "sink":
        # weight on position 0 and on the positions that repeat its token (vocabularies shorter than the run)
        toks = np.array(teacher_tokens(n, abs(shape[5])))
        w0 = min(float(np.min(p[:, toks[:pos + 1] == toks[0]].sum(axis=1)))
                 for pos, p in run.probs[0].items() if pos >= 1)
        assert w0 > 0.99, w0
        return {"min_weight_on_sink": w0}
    if kind == "outliers":
        ratio = min(float(np.max(np.abs(x)) / np.median(np.abs(x))) for x in run.resid.values())
        assert ratio >= 100, ratio
        return {"outlier_ratio": ratio}
    if kind == "loud":
        span = min(float(np.ptp(z)) for z in run.logits.values())
        toks = teacher_tokens(n + 1, abs(shape[5]))
        lp = min(float(ref64.log_softmax(z)[toks[p + 1]]) for p, z in run.logits.items() if p + 1 < n)
        assert span >= 40, span
        assert lp < -30, lp
        return {"logit_span": span, "min_target_logprob": lp}
    raise ValueError(kind)


def rel(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(np.asarray(a, dtype=np.float64) - b)) / (np.max(np.abs(b)) + 1e-30))


def compare_oracle(oracle, shape, data, n, check, tol=ORACLE_TOL):
    """Strict oracle vs ref64: logits at the check positions, the KV caches after position n-1."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint(shape, data)
    run = ref64.forward(shape, data, teacher_tokens(n, ck.vocab_size), check)
    logits, kc, vc = oracle_run(oracle, ck, n, check)
    for p in check:
        assert rel(logits[p], run.logits[p]) <= tol, (p, rel(logits[p], run.logits[p]))
    for got, want in ((kc, run.key_cache), (vc, run.value_cache)):
        assert rel(got, want.reshape(-1)) <= tol
    return run


@pytest.mark.parametrize("name", list(MODELS))
def test_oracle_vs_ref64_models(l2b, oracle, name):
    shape, _, n, check, _ = MODELS[name]
    compare_oracle(oracle, shape, payload(l2b, name).data, n, check)


@pytest.mark.parametrize("name", CPU_ENVELOPE)
def test_oracle_vs_ref64_envelope(oracle, name):
    shape, seed, n, check = ENVELOPE[name][:4]
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint(shape)
    data = oracle.synth_checkpoint(oracle.make_config(*ck.shape_tuple), ck.shared_weights, seed)
    compare_oracle(oracle, shape, data, n, check)


@pytest.mark.parametrize("kind", STRESS_KINDS)
@pytest.mark.parametrize("name", STRESS_MODELS)
def test_oracle_vs_ref64_stress(l2b, oracle, name, kind):
    shape, data = stress(l2b, name, kind)
    _, _, n, check, _ = MODELS[name]
    run = compare_oracle(oracle, shape, data, n, check)
    stress_check(kind, shape, run, n)


def test_payload_layout_matches_checkpoint_size(l2b):
    """ref64's own layout ends where the library's payload size does, for both classifier kinds."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    for shape in [MODELS["S"][0], MODELS["110M"][0], ENVELOPE["mqa64"][0]]:
        ck = shape_checkpoint(shape)
        assert ref64.payload_floats(shape) == l2b.checkpoint_floats(ck), shape


def test_ref64_agrees_with_numpy_restatement(l2b, stories15m):
    """The two float64 restatements (this one and test_independent_restatement.NumpyLlama) agree on
    stories15M to float64 rounding."""
    from test_independent_restatement import NumpyLlama
    ck = l2b.read_checkpoint(stories15m, mmap=False)
    toks = teacher_tokens(40, ck.vocab_size)
    check = (0, 1, 17, 39)
    run = ref64.forward(ck.shape_tuple[:5] + (ck.vocab_size if ck.shared_weights else -ck.vocab_size,
                                              ck.seq_len), np.asarray(ck.data), toks, check)
    m = NumpyLlama(ck)
    for pos, tok in enumerate(toks):
        lg = m.forward(tok, pos)
        if pos in check:
            assert rel(run.logits[pos], lg) <= 1e-6, pos     # differ only in the f32 RoPE angle
