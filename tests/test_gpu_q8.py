"""GPU: q8 device weights (int8 codes, one fp32 scale per 64 weights of a row).  A q8 context of a
payload P returns exactly what an fp32 context of dq(P) returns, on every kernel the library selects;
dq(P) is P with every matrix weight replaced by its dequantized value fl(q * s).

Each q8 kernel is the fp32 kernel the shape selects (the selection rules are computed at 4 bytes per
weight for every format), with W = q8: the same columns per thread, each weight rebuilt as fl(q * s) with
the scale of its absolute column, the same accumulators and reduction order.  So the check is bitwise
against an fp32 context of the dequantized payload, under the cases of test_gpu_variants.CASES (the
default and every launch switch of S and B, W, 110M and the head-size family):

  q8 instantiation                                       run by
  gemv_kernel<TPR, STORE | ARGMAX | QKV | SILU | RESID>  test_twin[S-default], [hs*-default], [S-nofuse]
  gemv8_kernel<every epilogue>                           test_twin[S-all-streaming-ldg], [B-ldg], [W-default]
  gemv_tma_kernel<every epilogue> (4-row x 4-step slots, test_twin[B-default], [S-all-streaming] (n = 772:
  16 KB of codes + 1 KB of scales)                       short last group, a row's last slot of one step),
                                                         [B-tma-stages2]
  prefill_gemm_kernel<QKV | SILU | RESID, 4>, <RESID, 2> test_twin[B-default] (prefill), test_batched[B]
  prefill_gemm_kernel<STORE | ARGMAX, 4>                 test_batched[B] (the batched classifier)
  attn_wo_kernel<NF> (scale index from the head's        test_twin[S-default], [hs*-default], [110M-fuse1]
  absolute column)
  layer-0 embedding row, dequantized (single / batched)  every test_twin case / test_batched[B]
  classifier aliasing a q8 embedding                     test_twin[110M-fuse1] (shared weights)
  synth_fill_q8_kernel                                   test_synthetic_equals_quantized_upload
"""
import dataclasses

import numpy as np
import pytest

from test_gpu_transformer import teacher_tokens
from test_gpu_variants import CASES, MODELS, l2b_env, payload
from test_q8_abi import dequant_matrices, matrix_shapes

pytestmark = pytest.mark.gpu

_dq = {}


def dequantized(l2b, name):
    """dq(P) of a test_gpu_variants model, and how many matrix weights the quantization changed."""
    if name not in _dq:
        ck = payload(l2b, name)
        data, n = dequant_matrices(l2b, ck, ck.data)
        _dq[name] = (dataclasses.replace(ck, data=data), n)
    return _dq[name]


def _eq(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    same = a.view(np.uint32) == b.view(np.uint32) if a.dtype == np.float32 else a == b
    assert same.all(), f"{what}: {int((~same).sum())} of {a.size} differ"


def twin_pair(l2b, name, env=None):
    ck, rk = payload(l2b, name), dequantized(l2b, name)[0]
    with l2b_env(env or {}):
        b = l2b.Transformer(ck, weight_format="q8")
        f = l2b.Transformer(rk)
    return b, f


@pytest.mark.parametrize("name,case,env", [(m, c, e) for m, c, e, _ in CASES],
                         ids=[f"{m}-{c}" for m, c, _, _ in CASES])
def test_twin(l2b, name, case, env):
    _, _, n, check, n_prompt = MODELS[name]
    b, f = twin_pair(l2b, name, env)
    with b, f:
        assert b.weight_info()[0] == "q8" and f.weight_info() == ("f32", 0)
        toks = teacher_tokens(n, b.ck.vocab_size)
        for pos, tok in enumerate(toks):                 # teacher-forced over the model's whole run
            lb, lf = b.forward(tok, pos), f.forward(tok, pos)
            if pos in check:
                _eq(lb, lf, f"logits at {pos}")
        for s in ("key_cache", "value_cache", "x"):
            _eq(b.state(s), f.state(s), s)
        for pos in check[:3]:
            assert b.forward_argmax(toks[pos], pos) == f.forward_argmax(toks[pos], pos)
        b.reset(); f.reset()
        forced = np.array(toks[1:9], np.int32)
        forced = np.concatenate([forced, np.full(8, -1, np.int32)])
        _eq(b.generate_argmax(toks[0], 0, 16, forced=forced, stop_on_bos=False),
            f.generate_argmax(toks[0], 0, 16, forced=forced, stop_on_bos=False), "generate_argmax")
        b.reset(); f.reset()
        _eq(b.prefill(toks[:n_prompt]), f.prefill(toks[:n_prompt]), "prefill logits")
        _eq(b.state("key_cache"), f.state("key_cache"), "prefill key cache")
        pb, cb = b.forward_sample(toks[n_prompt], n_prompt, 0.8, 0.9)
        pf, cf = f.forward_sample(toks[n_prompt], n_prompt, 0.8, 0.9)
        _eq(pb, pf, "forward_sample probs")
        assert (cb is None) == (cf is None) and (cb is None or np.array_equal(cb, cf))
        b.reset(); f.reset()
        lpb, gb = b.score(toks[:n_prompt])
        lpf, gf = f.score(toks[:n_prompt])
        _eq(lpb, lpf, "score log-probs")
        _eq(gb, gf, "score greedy")


@pytest.mark.parametrize("name", ["S", "B"])
def test_batched(l2b, name):
    b, f = twin_pair(l2b, name)
    with b, f:
        V = b.ck.vocab_size
        toks = teacher_tokens(40, V)
        sb = [b.session() for _ in range(4)]
        sf = [f.session() for _ in range(4)]
        try:
            for i in range(4):                           # sessions at different positions
                sb[i].prefill(toks[:3 + i], want_logits=False)
                sf[i].prefill(toks[:3 + i], want_logits=False)
            pos = [3, 4, 5, 6]
            t4 = toks[10:14]
            _eq(l2b.forward_batch(sb, t4, pos), l2b.forward_batch(sf, t4, pos), "forward_batch")
            pos = [p + 1 for p in pos]
            _eq(l2b.forward_argmax_batch(sb, t4, pos), l2b.forward_argmax_batch(sf, t4, pos), "argmax_batch")
            pos = [p + 1 for p in pos]
            rb = l2b.forward_sample_batch(sb, t4, pos, [1.0, 0.7, 1.0, 0.5], [0.9, 1.0, 0.95, 0.5])
            rf = l2b.forward_sample_batch(sf, t4, pos, [1.0, 0.7, 1.0, 0.5], [0.9, 1.0, 0.95, 0.5])
            _eq(rb[0], rf[0], "sample_batch probs")
            _eq(rb[2], rf[2], "sample_batch n_cand")
            pos = [p + 1 for p in pos]
            runs = [toks[0:1], toks[1:6], toks[6:9], toks[9:11]]     # NB 4 and NB 2 passes
            _eq(l2b.forward_ragged(sb, runs, pos), l2b.forward_ragged(sf, runs, pos), "forward_ragged")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            _eq(l2b.forward_argmax_ragged(sb, runs, pos), l2b.forward_argmax_ragged(sf, runs, pos), "argmax_ragged")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            rb = l2b.forward_sample_ragged(sb, runs, pos, [1.0] * 4, [0.9] * 4)
            rf = l2b.forward_sample_ragged(sf, runs, pos, [1.0] * 4, [0.9] * 4)
            _eq(rb[0], rf[0], "sample_ragged probs")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            gb = l2b.generate_argmax_batch(sb, t4, pos, 6, stop_on_bos=False)
            gf = l2b.generate_argmax_batch(sf, t4, pos, 6, stop_on_bos=False)
            for x, y in zip(gb, gf):
                _eq(x, y, "generate_argmax_batch")
            pos = [p + 6 for p in pos]
            vruns = [[int(g[-1])] + list(toks[20:23]) for g in gb]
            vb = l2b.verify_argmax_ragged(sb, vruns, pos)
            vf = l2b.verify_argmax_ragged(sf, vruns, pos)
            _eq(vb[1], vf[1], "n_accept")
            for x, y in zip(vb[0], vf[0]):
                _eq(x, y, "verify tokens")
            pos = [p + int(a) + 1 for p, a in zip(pos, vb[1])]
            wb = l2b.verify_sample_ragged(sb, vruns, pos, [1.0] * 4, [0.9] * 4)
            wf = l2b.verify_sample_ragged(sf, vruns, pos, [1.0] * 4, [0.9] * 4)
            _eq(wb[0], wf[0], "verify_sample probs")
            _eq(wb[2], wf[2], "verify_sample n_cand")
            for s in ("key_cache", "value_cache"):
                for x, y in zip(sb, sf):
                    _eq(x.state(s), y.state(s), f"session {s}")
            l2b.fork(sb[0], sb[1:], 5)
            l2b.fork(sf[0], sf[1:], 5)
            _eq(l2b.forward_batch(sb[1:], toks[30:33], [5, 5, 5]),
                l2b.forward_batch(sf[1:], toks[30:33], [5, 5, 5]), "after fork")
        finally:
            for s in sb + sf:
                s.close()


@pytest.mark.parametrize("name", ["S", "B"])
def test_speculative_q8_draft(l2b, name):
    """An fp32 target with a q8 draft of another seed: the tokens are the fp32 greedy loop's."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = payload(l2b, name)
    dk = shape_checkpoint(MODELS[name][0])
    dk.data = l2b.synth_checkpoint_host(dk, MODELS[name][1] + 1000)
    with l2b.Transformer(ck) as t, l2b.Transformer(dk, weight_format="q8") as d, l2b.Transformer(ck) as ref:
        want = ref.generate_argmax(1, 0, 24, stop_on_bos=False)
        got, _ = t.generate_speculative(d, 1, 0, 24, 3, stop_on_bos=False)
        _eq(got, want, "speculative tokens")


@pytest.mark.parametrize("name", ["S", "B"])
def test_dequantized_payload_and_counts(l2b, oracle, name):
    """dq(P): q8 of it changes nothing (n = 0) and is bitwise the fp32 context of dq(P); P: the count is
    numpy's; the fp32 context of dq(P) is within 1e-4 of the oracle of dq(P)."""
    ck, (rk, n) = payload(l2b, name), dequantized(l2b, name)
    with l2b.Transformer(rk, weight_format="q8") as b, l2b.Transformer(rk) as f, \
            l2b.Transformer(ck, weight_format="q8") as b0:
        assert b.weight_info() == ("q8", 0)
        want = int((matrix_view(ck, ck.data).view(np.uint32) != matrix_view(ck, rk.data).view(np.uint32)).sum())
        assert n == want and b0.weight_info() == ("q8", want)
        om = oracle.OracleModel(oracle.make_config(*rk.shape_tuple), rk.data, rk.shared_weights, W=8, kind="strict")
        for pos, tok in enumerate(teacher_tokens(8, ck.vocab_size)):
            lb, lf, lo = b.forward(tok, pos), f.forward(tok, pos), om.forward(tok, pos)
            _eq(lb, lf, f"dequantized payload logits at {pos}")
            assert float(np.max(np.abs(lf - lo)) / np.max(np.abs(lo))) <= 1e-4
        om.close()


def matrix_view(ck, data):
    return np.concatenate([data[off:off + r * c] for off, r, c in matrix_shapes(ck)])


@pytest.mark.parametrize("name", ["S", "B"])
def test_synthetic_equals_quantized_upload(l2b, name):
    ck = payload(l2b, name)
    seed = MODELS[name][1]
    with l2b.Transformer(ck, synthetic_seed=seed, weight_format="q8") as s, \
            l2b.Transformer(ck, weight_format="q8") as u:
        assert s.weight_info() == u.weight_info()
        assert s.weight_info()[1] == dequantized(l2b, name)[1] > 0
        for pos, tok in enumerate(teacher_tokens(6, ck.vocab_size)):
            _eq(s.forward(tok, pos), u.forward(tok, pos), f"synthetic vs upload at {pos}")
        _eq(s.state("key_cache"), u.state("key_cache"), "key cache")


def q8_row_bytes(n):
    """w_pitch<q8>(n): n codes padded to 16 bytes, then ceil(n / 64) fp32 scales padded to 16 bytes."""
    return (n + 15) // 16 * 16 + (4 * ((n + 63) // 64) + 15) // 16 * 16


@pytest.mark.parametrize("name", ["S", "B"])
def test_bytes_count_q8(l2b, name):
    ck = payload(l2b, name)
    b, f = twin_pair(l2b, name)
    with b, f:
        rb = q8_row_bytes
        d, h, L, V = ck.dim, ck.hidden_dim, ck.n_layers, ck.vocab_size
        kvd = d // ck.n_heads * ck.n_kv_heads
        mat = L * (d * rb(d) + 2 * kvd * rb(d) + d * rb(d) + 2 * h * rb(d) + d * rb(h)) + rb(d) + V * rb(d)
        wb, kb = b.step_bytes(3)
        wf, kf = f.step_bytes(3)
        assert wb == mat + 4 * 2 * L * d and kb == kf
        stored = (V * rb(d) + L * (2 * d * rb(d) + 2 * kvd * rb(d) + 2 * h * rb(d) + d * rb(h))
                  + (0 if ck.shared_weights else V * rb(d)))
        _, ub = b.load_stats()
        assert ub == stored + 4 * (2 * L * d + d)
        per_layer = {"qkv_rope": (d + 2 * kvd) * rb(d), "wo": d * rb(d), "w13_silu": 2 * h * rb(d),
                     "w2": d * rb(h), "classifier": V * rb(d)}
        prof = b.profile_step(1, 0)
        seen = set()
        for n, l, _, by in prof:
            if n in per_layer:
                assert by == per_layer[n], (n, l, by, per_layer[n])
                seen.add(n)
        assert seen >= {"w13_silu", "w2", "classifier"}, seen
