"""GPU: every kernel instantiation and launch mode the library can select, not only the defaults.

The library picks among many kernel instantiations at run time: by shape (`launch_gemv`,
`pick_attention`, `pick_attn_wo`, `pf_prepare` in csrc/llama2_b200.cu) and by the L2B_* switches
that `create_rank` reads from the environment when a context is created.  Every case below creates
a context under one environment and runs the same checker on it:

  * `forward` teacher-forced over the whole run, logits within 1e-4 relative of the strict oracle at
    the model's check positions, and the key/value cache after the last step;
  * `forward_argmax` at the check positions == the first-index `np.argmax` of that position's
    `forward` logits (the reference's strict '>' tie rule, src/main.zig:715-726);
  * `generate_argmax` with a forced prefix, then free-running steps == a host loop of `forward_argmax`;
  * one `forward_sample` step: probabilities within 1e-4 of the exact float64 softmax of the step's
    logits, candidates == the host filter (or, past the candidate capacity, their negated count);
  * `prefill` == token-by-token `forward`: bit for bit (include/llama2_b200.h), 1e-6 on the batched
    kernel of bandwidth-bound shapes (prefill_gemm_kernel, csrc/l2b_device.cuh), like
    test_batched_prefill_on_bandwidth_bound_shapes.

Switches that change neither the kernels' arithmetic nor their summation order must also reproduce
the default context's logits and caches bit for bit (`BITWISE`).  The oracle runs once per model.

Ledger: kernel instantiation -> a test that runs it (ids relative to this module unless named)
  gemv_kernel<TPR, STORE | ARGMAX | QKV | SILU | RESID>   test_variant[S-default] (TPR 16/32),
                                                         test_variant[B-latency-tpr8] (TPR 8),
                                                         test_variant[hs4-default] (TPR 8, n = 32)
  gemv8_kernel<QKV | SILU | ARGMAX> (fused rmsnorm, dim > 5760)   test_variant[W-default]
  gemv8_kernel<every epilogue>                            test_variant[B-ldg], test_variant[S-all-streaming-ldg]
  gemv_tma_kernel<QKV | SILU | ARGMAX | STORE | RESID>     test_variant[B-default], test_variant[S-all-streaming]
  gemv_tma_kernel ring depth 2, 2 CTAs/SM, 1 stage before the wait   test_variant[B-tma-stages2-ctas2],
                                                         test_variant[B-tma-prefill1]
  gemv_*<EPI_XCHG>                                        tensor parallel only: tests/test_gpu_tp.py
  device argmax: ties across CTAs, all-negative logits, last (half-empty) row pair of an odd vocabulary
                                                         test_device_argmax_edges[*]
  attention_flash_kernel<1> LPR 1 / LPR 2                 test_variant[hs4-nofuse] / test_variant[hs8-nofuse]
  attention_flash_kernel<2>                               test_variant[B-default] (GQA, head_size 64)
  attention_flash_kernel<3> LPR 1 / 2 / 4                 test_variant[hs12-nofuse] / [hs24-nofuse] / [S-nofuse]
  attention_flash_kernel<4>                               test_variant[W-default], test_variant[hs128-nofuse]
  attention_flash_kernel<5>, <6>, <8>                     test_variant[hs20-nofuse], [hs192-nofuse], [hs256-nofuse]
  attention_flash_kernel, 32 timeline splits              test_variant[S-attn-min-chunk8]
  attention_kernel (3-pass) incl. its split merge         test_variant[hs28-default], [hs72-default],
                                                         [hs224-default] (selected by shape), [S-attn-3pass],
                                                         [B-attn-3pass]; test_gpu_ops.py::test_attention_head_kernels_vs_oracle
  attn_wo_kernel<1>, <3>, <5>, <6>, <8>                   test_variant[hs4-default] / [S-default] / [hs20-default] /
                                                         [hs192-default] / [hs256-default]
  attn_wo_kernel<2>, <4>                                  test_variant[110M-fuse1] / [hs128-default]
  attn_wo_kernel cluster sizes 1, 2, 4 (default 8)        test_variant[S-attn-r1], [S-attn-r2], [S-attn-r4]
  prefill_gemm_kernel<QKV | SILU | RESID, NB 4 and 2> with GQA (the TMA stream code of gemv_tma_kernel
  with NB vectors)                                        test_variant[B-default] (prefill check),
                                                         test_variant[S-all-streaming] (head_size 48)
  position-by-position device prefill loop               test_variant[B-prefill-batch0] and every small model
  eager launches / launches without PDL                  test_variant[*-no-graph], [*-no-pdl], [*-no-graph-no-pdl]
  sample_prep_kernel past the candidate capacity          test_sampler_candidate_overflow

At the resource limits (tests/test_gpu_envelope.py, ids relative to test_envelope):
  gemv_tma_kernel, fused rmsnorm with all 5 gain slices    [dim5760-default], [llama2-13B-default]
  gemv8_kernel<QKV | SILU | ARGMAX> just past them         [dim5888-default], [llama2-70B-default] (dim 8192)
  gemv_tma_kernel ring depth 2 / 3 chosen by the budget    [w2-hid41216-default] / [pf-hid28672-default],
                                                         [llama2-70B-default]
  gemv8_kernel<RESID> with the whole shared memory as x     [x-hid57600-default]; one float more:
                                                         test_envelope_refused_at_create[x-hid57604]
  prefill_gemm_kernel<*, 4> at 4 ring stages, <RESID, 2> at 2   [dim5760-default], [pf-hid19840-default]
  position-loop prefill past the NB = 2 budget            [pf-hid19844-default], [pf-hid28672-default]
  attention_flash_kernel / attention_kernel / attn_wo_kernel, splits longer than min_chunk
                                                         [ctx4096-h32-*], [ctx16384-h1-*]
  attention_kernel at the longest accepted context        [ctx1605632-attn-3pass]
  single-CTA grids, odd last row pair, kv_mul 64          [vocab1-*], [vocab2-seq1-*], [vocab3-2layers-*], [mqa64-*]
  sample_prep_kernel over 128256 entries                  [llama3-8B-default]
"""
import contextlib
import os

import numpy as np
import pytest

from test_gpu_transformer import REL_TOL, rel_err, teacher_tokens

pytestmark = pytest.mark.gpu

# name -> shape (dim, hidden, layers, heads, kv_heads, vocab (negative: unshared classifier), seq_len),
# synthetic seed, positions run, positions checked, prompt length of the prefill check
MODELS = {
    # latency kernels, attention+wo fused by default; GQA (kv_mul 3), hidden/4 odd, odd unshared
    # classifier, a context that crosses the 256-position attention split
    "S": ((288, 772, 2, 6, 2, -1001, 300), 31, 300, (0, 1, 2, 100, 255, 256, 257, 299), 258),
    # TinyLlama's layer shape, 2 layers: TMA ring, batched prefill with GQA, odd vocabulary through
    # the TMA argmax
    "B": ((2048, 5632, 2, 32, 4, -32003, 600), 32, 260, (0, 1, 2, 127, 255, 256, 257, 259), 258),
    # dim > 5760: the fused-rmsnorm GEMVs leave the TMA ring for gemv8_kernel
    "W": ((6144, 2048, 1, 48, 8, -1000, 64), 33, 64, (0, 1, 2, 31, 63), 32),
    # stories110M shape, 2 layers (L2B_FUSE=1 runs attn_wo_kernel<2> at dim 768)
    "110M": ((768, 2048, 2, 12, 12, 32000, 1024), 110, 40, (0, 1, 2, 20, 39), 21),
}

# head-size family: small GQA / MQA models over ~520 positions (two attention splits crossed)
HEAD_SIZES = {4: (8, 2), 8: (8, 1), 12: (4, 2), 20: (4, 1), 24: (4, 2), 128: (4, 2), 192: (2, 1),
              256: (2, 1), 28: (4, 2), 72: (4, 2), 224: (2, 1)}       # head_size -> (heads, kv_heads)
for _hs, (_h, _kv) in HEAD_SIZES.items():
    MODELS[f"hs{_hs}"] = ((_hs * _h, 2 * _hs * _h + 4, 2, _h, _kv, -97, 520), 40 + _hs, 520,
                          (0, 1, 255, 256, 257, 511, 512, 513, 519), 258)


def _flash_nf(hs):
    """NF of attention_flash_kernel / attn_wo_kernel for head_size hs, or None (3-pass kernel only)."""
    hs4 = hs // 4
    lpr = 8 if hs4 % 8 == 0 else 4 if hs4 % 4 == 0 else 2 if hs4 % 2 == 0 else 1
    nf = hs4 // lpr
    return nf if nf in (1, 2, 3, 4, 5, 6, 8) else None


ALL_STREAMING = {"L2B_BIG_MIN_N": "4", "L2B_GEMV8_MIN_BYTES": "0", "L2B_FUSE": "0"}

# Switches that must reproduce the default context bit for bit: graphs, PDL, step timing and the
# upload chunking do not touch the arithmetic, and the TMA ring's per-row summation order (lane
# columns, butterfly, warps in fixed order) is the same for every ring depth and grid size.
BITWISE = {
    "no-graph": {"L2B_NO_GRAPH": "1"},
    "no-pdl": {"L2B_NO_PDL": "1"},
    "no-graph-no-pdl": {"L2B_NO_GRAPH": "1", "L2B_NO_PDL": "1"},
    "tma-stages2": {"L2B_TMA_STAGES": "2"},
    "tma-ctas2": {"L2B_TMA_CTAS": "2"},
    "tma-stages2-ctas2": {"L2B_TMA_STAGES": "2", "L2B_TMA_CTAS": "2"},   # small ring: 2 CTAs fit per SM
    "tma-prefill1": {"L2B_TMA_PREFILL": "1"},
    "time-steps": {"L2B_TIME_STEPS": "1"},
    "stage-1mb": {"L2B_STAGE_MB": "1"},           # the pinned upload of B takes ~900 chunks
}

CASES = []                                        # (model, case name, env, compare bitwise with default)
for _m in ("S", "B"):
    CASES.append((_m, "default", {}, False))
    CASES += [(_m, k, v, True) for k, v in BITWISE.items()]
    CASES += [(_m, "ldg", {"L2B_GEMV_BIG": "ldg"}, False),
              (_m, "latency-only", {"L2B_GEMV8_MIN_BYTES": "-1"}, False)]
CASES += [
    # every GEMV on the TMA ring (and on gemv8), every epilogue, at dim 288; fusion off because
    # launch_gemv refuses the partial-vector prologue on the streaming kernels
    ("S", "all-streaming", ALL_STREAMING, False),
    ("S", "all-streaming-ldg", dict(ALL_STREAMING, L2B_GEMV_BIG="ldg"), False),
    # fusion on S would bypass the stand-alone attention kernel, so these turn it off
    ("S", "attn-3pass", {"L2B_FUSE": "0", "L2B_ATTN": "3pass"}, False),
    ("S", "attn-min-chunk8", {"L2B_FUSE": "0", "L2B_ATTN_MIN_CHUNK": "8"}, False),   # 32 timeline splits
    ("S", "nofuse", {"L2B_FUSE": "0"}, False),
    ("S", "prefill-batch0", {"L2B_PREFILL_BATCH": "0"}, False),
    ("S", "attn-r1", {"L2B_ATTN_R": "1"}, False),
    ("S", "attn-r2", {"L2B_ATTN_R": "2"}, False),
    ("S", "attn-r4", {"L2B_ATTN_R": "4"}, False),
    ("B", "attn-3pass", {"L2B_ATTN": "3pass"}, False),
    ("B", "attn-min-chunk8", {"L2B_ATTN_MIN_CHUNK": "8"}, False),
    ("B", "prefill-batch0", {"L2B_PREFILL_BATCH": "0"}, False),
    # the classifier's 32003 rows on the latency kernel: threads per row shrink down to 8
    ("B", "latency-tpr8", {"L2B_GEMV8_MIN_BYTES": "-1", "L2B_TPR_TILES": "1"}, False),
    ("W", "default", {}, False),
    ("110M", "fuse1", {"L2B_FUSE": "1"}, False),
]
for _hs in HEAD_SIZES:
    CASES.append((f"hs{_hs}", "default", {}, False))
    if _flash_nf(_hs) is not None:                # the default fuses attention+wo: run the stand-alone kernel too
        CASES.append((f"hs{_hs}", "nofuse", {"L2B_FUSE": "0"}, False))


@contextlib.contextmanager
def l2b_env(env):
    """Exactly the L2B_* variables of `env` for the contexts created inside (read at creation)."""
    saved = {k: v for k, v in os.environ.items() if k.startswith("L2B_")}
    for k in saved:
        del os.environ[k]
    os.environ.update(env)
    try:
        yield
    finally:
        for k in [k for k in os.environ if k.startswith("L2B_")]:
            del os.environ[k]
        os.environ.update(saved)


PF_SMEM_BUDGET = 227 * 1024 - 8192               # kPfSmemBudget: dynamic shared memory of prefill_gemm_kernel
TMA_STAGE_BYTES = 8 * 256 * 16                   # one ring stage: 8 rows x 256 float4


def batched_prefill(shape, env):
    """Whether l2b_prefill takes the batched kernel under `env` (the shape test of pf_prepare)."""
    dim, hid, _, heads = shape[:4]
    if env.get("L2B_PREFILL_BATCH", "1").startswith("0") or env.get("L2B_ATTN") == "3pass":
        return False
    big_min_n = int(env.get("L2B_BIG_MIN_N", "1024"))
    big_min_n = big_min_n if big_min_n >= 4 else 1024
    min_bytes = int(env.get("L2B_GEMV8_MIN_BYTES", str(8 << 20)))
    return (dim >= big_min_n and hid >= big_min_n and dim <= 5760 and 0 <= min_bytes <= dim * dim * 4
            and _flash_nf(dim // heads) is not None
            # a ring of >= 2 stages next to 4 dim-wide inputs (qkv, wo, w13) and 2 hidden-wide ones (w2)
            and 4 * dim * 4 + 2 * TMA_STAGE_BYTES <= PF_SMEM_BUDGET
            and 2 * hid * 4 + 2 * TMA_STAGE_BYTES <= PF_SMEM_BUDGET)


def prefill_launches(shape, env, n_tokens, step_launches):
    """Kernels one logits-free l2b_prefill of n_tokens launches: per layer and chunk of 4 positions the
    batched path runs qkv, attention, wo, w13 and one w2 per pair of positions; the position loop
    runs one decode step (without the classifier, plus the token advance) per position."""
    if not batched_prefill(shape, env):
        return n_tokens * step_launches
    chunks = [min(4, n_tokens - i) for i in range(0, n_tokens, 4)]
    return shape[2] * sum(4 + (nb + 1) // 2 for nb in chunks)


_payloads, _refs, _defaults = {}, {}, {}


def payload(l2b, name):
    if name not in _payloads:
        from llama2_zig_b200.checkpoint import shape_checkpoint
        shape, seed = MODELS[name][:2]
        ck = shape_checkpoint(shape)
        ck.data = l2b.synth_checkpoint_host(ck, seed)
        _payloads[name] = ck
    return _payloads[name]


def oracle_run(oracle, ck, n, check):
    """Strict-oracle logits at the check positions of a teacher-forced run of n positions, and the KV
    caches after the last position."""
    om = oracle.OracleModel(oracle.make_config(*ck.shape_tuple), ck.data, ck.shared_weights, W=8, kind="strict")
    logits = {}
    for pos, tok in enumerate(teacher_tokens(n, ck.vocab_size)):
        lg = om.forward(tok, pos)
        if pos in check:
            logits[pos] = lg
    ref = (logits, om.state("key_cache"), om.state("value_cache"))
    om.close()
    return ref


def oracle_ref(l2b, oracle, name):
    """oracle_run of a model of MODELS (once per model)."""
    if name not in _refs:
        _, _, n, check, _ = MODELS[name]
        _refs[name] = oracle_run(oracle, payload(l2b, name), n, check)
    return _refs[name]


def softmax64(x):
    e = np.exp(x.astype(np.float64) - np.max(x))
    return e / e.sum()


def host_candidates(probs, top_p):
    cutoff = np.float32((np.float32(1.0) - np.float32(top_p)) / (np.float32(probs.size) - np.float32(1.0)))   # :761
    return np.nonzero(probs >= cutoff)[0]


def run_case(l2b, oracle, name, env):
    """Create a context under `env`, run every checker on it, return (logits by position, kcache, vcache)."""
    _, _, n, check, n_prompt = MODELS[name]
    return check_context(l2b, payload(l2b, name), n, check, n_prompt, oracle_ref(l2b, oracle, name), env)


def check_context(l2b, ck, n, check, n_prompt, ref, env):
    """Every checker on a context of checkpoint `ck` created under `env`: n teacher-forced positions
    against ref = oracle_run(.., n, check), prefill of the first n_prompt tokens (n_prompt - 1 in
    check).  Returns (logits by position, kcache, vcache)."""
    want, kref, vref = ref
    toks = teacher_tokens(n, ck.vocab_size)
    kv = ck.seq_len * (ck.dim // ck.n_heads) * ck.n_kv_heads          # floats per layer of one cache
    with l2b_env(env), l2b.Transformer(ck) as t:
        got = {}
        for pos, tok in enumerate(toks):
            lg = t.forward(tok, pos)
            if pos in check:
                got[pos] = lg
                assert rel_err(lg, want[pos]) <= REL_TOL, (pos, rel_err(lg, want[pos]))
        _, step_launches = t.last_timing()
        kc, vc = t.state("key_cache"), t.state("value_cache")
        np.testing.assert_allclose(kc, kref, rtol=0, atol=1e-4 * np.max(np.abs(kref)))
        np.testing.assert_allclose(vc, vref, rtol=0, atol=1e-4 * np.max(np.abs(vref)))

        # device argmax (re-running a position is idempotent) == first-index argmax of the logits
        for pos in check:
            assert t.forward_argmax(toks[pos], pos) == int(np.argmax(got[pos])), pos

        # one sampler step on the last checked position; a single-entry vocabulary is refused
        p = check[-1]
        if ck.vocab_size < 2:
            with pytest.raises(l2b.L2BError) as e:
                t.forward_sample(toks[p], p, 1.0, 0.9)
            assert e.value.status == -1
        else:
            probs, cand, n_cand = t.forward_sample(toks[p], p, 1.0, 0.9, with_count=True)
            ref = softmax64(got[p])
            assert np.max(np.abs(probs - ref)) <= 1e-4 * np.max(ref)
            keep = host_candidates(probs, 0.9)
            if keep.size <= 8192:
                assert n_cand == keep.size and np.array_equal(cand["index"], keep.astype(np.int32))
                assert np.array_equal(cand["prob"], probs[keep])
            else:
                assert n_cand == -keep.size and cand is None

        # on-device loop: 4 forced steps, then free-running ones (12 in all, or up to seq_len) ==
        # host loop of forward_argmax
        steps = min(12, ck.seq_len)
        gen = teacher_tokens(steps + 1, ck.vocab_size)
        forced = np.full(steps, -1, np.int32)
        forced[:4] = gen[1:min(5, steps + 1)]
        t.reset()
        out = t.generate_argmax(gen[0], 0, steps, forced=forced, stop_on_bos=False)
        t.reset()
        host, tok = [], gen[0]
        for pos in range(steps):
            nxt = t.forward_argmax(tok, pos)
            tok = int(forced[pos]) if forced[pos] >= 0 else nxt
            host.append(tok)
        assert out.tolist() == host

        # which path l2b_prefill takes (batched kernel or position loop): its launch count
        if n_prompt > 1:
            t.reset()
            t.prefill(toks[:n_prompt - 1], 0, want_logits=False)
            assert t.last_timing()[1] == prefill_launches(ck.shape_tuple, env, n_prompt - 1, step_launches)

        # prefill of the first n_prompt teacher tokens == the token-by-token logits and KV rows
        t.reset()
        lp = t.prefill(toks[:n_prompt], 0)
        kp, vp = t.state("key_cache"), t.state("value_cache")
        rows = n_prompt * kv // ck.seq_len
        exact = not batched_prefill(ck.shape_tuple, env)
        for l in range(ck.n_layers):
            sl = slice(l * kv, l * kv + rows)
            for a, b in ((kp[sl], kc[sl]), (vp[sl], vc[sl])):
                if exact:
                    assert np.array_equal(a, b), l
                else:
                    assert np.max(np.abs(a - b)) <= 1e-6 * np.max(np.abs(b)), l
        if exact:
            assert np.array_equal(lp, got[n_prompt - 1])
        else:
            assert rel_err(lp, got[n_prompt - 1]) <= 1e-6
    return got, kc, vc


def default_run(l2b, oracle, name):
    if name not in _defaults:
        _defaults[name] = run_case(l2b, oracle, name, {})
    return _defaults[name]


@pytest.mark.parametrize("name,case,env,bitwise", CASES, ids=[f"{m}-{c}" for m, c, _, _ in CASES])
def test_variant(l2b, oracle, name, case, env, bitwise):
    if case == "default":
        default_run(l2b, oracle, name)
        return
    got, kc, vc = run_case(l2b, oracle, name, env)
    if bitwise:
        ref, kref, vref = default_run(l2b, oracle, name)
        for pos in ref:
            assert np.array_equal(got[pos], ref[pos]), pos
        assert np.array_equal(kc, kref) and np.array_equal(vc, vref)


# ---------------------------------------------------------------------------------------------
# Device argmax edges on crafted classifiers (built like oracle_lib.bos_stop_payload: unshared
# classifier rows edited in the payload).  r is a random direction; every other row is scaled down
# so that the crafted rows hold the maximum.  GPU logits are the reference here: the device argmax
# must be their first-index argmax, and that must be the crafted row.
#   tie  : rows 5 and V-1 are r*8 (exact twins, first and last CTA), rows 6 and V-2 are -r*8; the
#          winner is 5 or 6 depending on the sign of r.xn, never its later twin.  Rows 5 and 6 sit
#          in the third and fourth row pair of the first tile.
#   neg  : row k is a_k * r with distinct positive, non-monotone a_k: all logits share the sign of
#          r.xn, so the largest a_k wins on one sign and the smallest on the other (all negative).
#   last : row V-1 (alone in the half-empty last row pair of an odd vocabulary) is r*8, row V-2 -r*8.
# ---------------------------------------------------------------------------------------------
EDGE_KERNELS = {"latency": ("S", {}), "tma": ("B", {}), "gemv8": ("B", {"L2B_GEMV_BIG": "ldg"})}


def crafted(l2b, name, kind):
    ck = payload(l2b, name)
    V, dim = ck.vocab_size, ck.dim
    data = ck.data.copy()
    wcls = data[data.size - V * dim:].reshape(V, dim)
    r = np.random.default_rng(7).standard_normal(dim).astype(np.float32) * np.float32(0.04)
    if kind == "neg":
        a = (0.5 + ((np.arange(V, dtype=np.int64) * 7919) % V) / V).astype(np.float32)
        wcls[:] = a[:, None] * r[None, :]
        return data, a
    wcls *= np.float32(0.01)
    if kind == "tie":
        wcls[5] = wcls[V - 1] = r * np.float32(8)
        wcls[6] = wcls[V - 2] = -r * np.float32(8)
    else:
        wcls[V - 1] = r * np.float32(8)
        wcls[V - 2] = -r * np.float32(8)
    return data, None


@pytest.mark.parametrize("kind", ["tie", "neg", "last"])
@pytest.mark.parametrize("kernel", list(EDGE_KERNELS))
def test_device_argmax_edges(l2b, kernel, kind):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    name, env = EDGE_KERNELS[kernel]
    data, a = crafted(l2b, name, kind)
    ck = shape_checkpoint(MODELS[name][0], data)
    V = ck.vocab_size
    toks = teacher_tokens(24, V)
    signs = set()
    with l2b_env(env), l2b.Transformer(ck) as t:
        for pos, tok in enumerate(toks):
            lg = t.forward(tok, pos)
            best = int(np.argmax(lg))
            assert t.forward_argmax(tok, pos) == best, pos
            if kind == "tie":
                assert best in (5, 6), (pos, best)
                assert lg[5] == lg[V - 1] and lg[6] == lg[V - 2]           # the twins really tie
            elif kind == "last":
                assert best in (V - 1, V - 2), (pos, best)
            elif np.all(lg > 0) or np.all(lg < 0):
                signs.add(bool(lg[0] > 0))
                assert best == (int(np.argmax(a)) if lg[0] > 0 else int(np.argmin(a))), pos
        if kind == "neg":
            assert signs == {True, False}, signs
        # free-running on-device loop == host loop of forward_argmax
        t.reset()
        out = t.generate_argmax(toks[0], 0, 16, stop_on_bos=False)
        t.reset()
        host, tok = [], toks[0]
        for pos in range(16):
            tok = t.forward_argmax(tok, pos)
            host.append(tok)
        assert out.tolist() == host
        if kind == "tie":
            assert V - 1 not in host and V - 2 not in host      # a later twin never wins


def test_sampler_candidate_overflow(l2b):
    """T = 4, top_p = 0.999 on B's 32003-entry vocabulary: more candidates pass the top-p prefilter
    than the device keeps (8192; about 23500 pass at this position, 3000 at T = 2), so
    l2b_forward_sample reports their negated count, which must be the host filter's count."""
    ck = payload(l2b, "B")
    toks = teacher_tokens(3, ck.vocab_size)
    with l2b_env({}), l2b.Transformer(ck) as t:
        for pos, tok in enumerate(toks[:-1]):
            t.forward(tok, pos)
        lg = t.forward(toks[-1], 2)
        probs, cand, n_cand = t.forward_sample(toks[-1], 2, 4.0, 0.999, with_count=True)
        scaled = (lg / np.float32(4.0)).astype(np.float32)
        assert np.max(np.abs(probs - softmax64(scaled))) <= 1e-4 * np.max(probs)
        keep = host_candidates(probs, 0.999)
        assert keep.size > 8192
        assert cand is None and n_cand == -keep.size
