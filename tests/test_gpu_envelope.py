"""GPU: every shape class the C ABI accepts, at each kernel's resource limit and just past it.

include/llama2_b200.h accepts any dim, hidden_dim and head_size that are multiples of 4 (head_size
<= 256).  Between those shapes the library picks kernels by shared-memory and register budgets it
computes at run time (`launch_gemv`, `pf_prepare` / `pf_launch`, the attention split set-up in
`create_rank`, csrc/llama2_b200.cu).  Each case here is a 1- or 2-layer synthetic checkpoint placed
on one side of such a limit, run through test_gpu_variants.check_context: teacher-forced logits and
KV cache against the strict oracle, device argmax, the on-device loop, one sampler step, prefill
against token-by-token `forward`, and which prefill path the library took (batched kernel or
position loop, from the launch count).  Shapes are (dim, hidden, layers, heads, kv_heads, vocab
(negative: unshared classifier), seq_len).

  limit                                   inside                       outside
  rmsnorm gain in the TMA ring's          dim5760: 5th register slice  dim5888: fused GEMVs on gemv8_kernel,
  registers (5 x 288 float4)              full, batched prefill with   prefill by position
                                          4 ring stages
  batched prefill, w2's 2 inputs next     pf-hid19840: exactly the     pf-hid19844: position loop;
  to a ring of >= 2 stages                budget, 2 stages             pf-hid28672: past the budget by more
                                                                       than the budget (the unsigned
                                                                       subtraction used to wrap and pick the
                                                                       batched kernel with a negative ring)
  TMA ring of >= 2 stages on w2's input   w2-hid41216: 2 stages        w2-hid41220: w2 on gemv8_kernel
  activation vector in shared memory      x-hid57600: w2 on gemv8      hid 57604: l2b_create refuses (-2)
                                          with all of it
  attention split longer than min_chunk   ctx4096-h32: 9 splits of 456 at the last position; ctx16384-h1:
                                          32 splits of 512 (flash); attn_wo's 8 cluster splits of 512 / 2048
  3-pass score buffer at create           ctx1605632: the longest      seq_len 1605633: refused (-2)
                                          accepted context, a few positions
  degenerate sizes                        vocab 1, 2, 3; dim = head_size = hidden = 4; seq_len 1 and 3;
                                          64 query heads on 1 kv head
  Llama-family layers                     llama2-13B, Llama-3-8B (GQA 4, 128256-entry vocabulary),
                                          llama2-70B (dim 8192 on gemv8_kernel, w2's ring 3 stages)

KV caches (test_envelope_kv): every (shape, environment) above, on device-synthesized weights of the same
seed, runs each KV pair bit for bit (KV_PAIRS): paged f32 == contiguous f32 (which test_envelope ties to
the oracle), bf16 == f32-round-bf16, paged bf16 == bf16, e4m3 == f32-round-e4m3 with unit and with stress
scales, paged e4m3 == e4m3 with stress scales.  Checked: logits at the checked positions, both caches
below the appended count, forward_argmax at the first 3 checked positions, generate_argmax (min(16,
seq_len) steps, half forced), prefill of the prompt (logits and rows), forward_sample at the prompt's end
(not on vocab 1: the sampler refuses it) and score of the prompt.  ctx4096-h32 and ctx16384-h1 prefill
to their last 8 positions and step those, then fork 4 sessions at seq_len - 70, - 64, - 33 and - 8 (page
offsets 58, 0, 31, 56) for one forward_batch and one forward_ragged of 3, 4, 2 and 1 tokens.  With stress
scales, a prefill of the rows they were set from (min(seq_len, 258)) equals its twin and holds >= 1 %
saturated K and >= 1 % subnormal V codes in layer 0, except on vocab1 and ctx1605632 (the teacher tokens
cycle through 1 or 3 tokens: V repeats its rows, and the smallest |V| is the 3 % quantile itself) and
vocab2-seq1 (one row of 4 values, none of which rounds to a subnormal code).  ctx1605632 has no paged pairs: past the paged limit.

Paged seq_len limits (test_paged_seq_len_limit; 1 layer, paged against a contiguous twin created after it
is closed, bit for bit: logits at positions 0..4, one forward_batch with a session at position 2, and both
caches' rows in use):
  tiny-1556832        (4, 4, 1, 1, 1, -3, 1556832): the longest paged context; 1556833 is refused (-2)
  hs256-891384/5      head size 256 x 2 heads, attn_wo_kernel<8>: 49,152 / 49,160 B, each side of the
                      48 KiB a kernel gets without opting in
  hs256-1556832       59,552 B, the paged limit at head size 256
  hs192-1448441       head size 192 x 2 heads, attn_wo_kernel<6>: 49,160 B, just past 48 KiB
  hs192-1558816       50,880 B, the paged limit at head size 192
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_variants import ALL_STREAMING, batched_prefill, check_context, oracle_run

pytestmark = pytest.mark.gpu


def _tail(n, k=8):
    return tuple(range(n - k, n))


FUSE0 = {"L2B_FUSE": "0"}
PASS3 = {"L2B_FUSE": "0", "L2B_ATTN": "3pass"}
LONG_ENVS = {"default": {}, "nofuse": FUSE0, "attn-3pass": PASS3}
TINY_ENVS = {"default": {}, "all-streaming": ALL_STREAMING}

# name -> shape, synthetic seed, positions run, positions checked, prompt length of the prefill
# check (its last position is checked), batched prefill under the default environment, environments
ENVELOPE = {
    "dim5760": ((5760, 2048, 1, 45, 9, -1000, 64), 51, 21, (0, 1, 2, 19, 20), 20, True, {"default": {}}),
    "dim5888": ((5888, 2048, 1, 46, 2, -1000, 64), 52, 21, (0, 1, 2, 19, 20), 20, False, {"default": {}}),
    "pf-hid19840": ((2048, 19840, 1, 16, 4, -1000, 64), 53, 21, (0, 1, 2, 19, 20), 20, True, {"default": {}}),
    "pf-hid19844": ((2048, 19844, 1, 16, 4, -1000, 64), 54, 21, (0, 1, 2, 19, 20), 20, False, {"default": {}}),
    "pf-hid28672": ((2048, 28672, 1, 16, 4, -1000, 64), 55, 21, (0, 1, 2, 19, 20), 20, False, {"default": {}}),
    "w2-hid41216": ((1024, 41216, 1, 8, 2, -1000, 64), 56, 12, (0, 1, 10, 11), 11, False, {"default": {}}),
    "w2-hid41220": ((1024, 41220, 1, 8, 2, -1000, 64), 57, 12, (0, 1, 10, 11), 11, False, {"default": {}}),
    "x-hid57600": ((1024, 57600, 1, 8, 2, -1000, 64), 58, 12, (0, 1, 10, 11), 11, False, {"default": {}}),
    # long contexts: the cache is filled by prefill up to the first of the last 8 positions
    "ctx4096-h32": ((256, 516, 1, 32, 8, -97, 4096), 59, 4096, _tail(4096), 4089, False, LONG_ENVS),
    "ctx16384-h1": ((32, 68, 1, 1, 1, -97, 16384), 60, 16384, _tail(16384), 16377, False, LONG_ENVS),
    "ctx1605632": ((4, 4, 1, 1, 1, -3, 1605632), 61, 6, (0, 1, 4, 5), 5, False, {"default": {}, "attn-3pass": PASS3}),
    # degenerate sizes
    "vocab1": ((4, 4, 1, 1, 1, -1, 3), 62, 3, (0, 1, 2), 3, False, TINY_ENVS),
    "vocab2-seq1": ((4, 4, 1, 1, 1, -2, 1), 63, 1, (0,), 1, False, TINY_ENVS),
    "vocab3-2layers": ((4, 4, 2, 1, 1, 3, 3), 64, 3, (0, 1, 2), 3, False, TINY_ENVS),
    "mqa64": ((256, 260, 1, 64, 1, -97, 40), 65, 40, (0, 1, 2, 20, 39), 21, False, TINY_ENVS),
    # real Llama-family layer shapes, one layer each
    "llama2-13B": ((5120, 13824, 1, 40, 40, -32000, 64), 66, 21, (0, 1, 2, 19, 20), 20, True, {"default": {}}),
    "llama3-8B": ((4096, 14336, 1, 32, 8, -128256, 64), 67, 21, (0, 1, 2, 19, 20), 20, True, {"default": {}}),
    "llama2-70B": ((8192, 28672, 1, 64, 8, -32000, 64), 68, 21, (0, 1, 2, 19, 20), 20, False, {"default": {}}),
}
SLOW = {"llama2-70B"}                         # ~6 GB of host payload

PARAMS = [pytest.param(name, env_name, marks=[pytest.mark.slow] if name in SLOW else [],
                       id=f"{name}-{env_name}")
          for name, spec in ENVELOPE.items() for env_name in spec[6]]

_last = {}                                    # one model's payload and oracle run at a time (parameters are grouped)


def model(l2b, oracle, name):
    if name not in _last:
        from llama2_zig_b200.checkpoint import shape_checkpoint
        _last.clear()
        shape, seed, n, check = ENVELOPE[name][:4]
        ck = shape_checkpoint(shape)
        ck.data = oracle.synth_checkpoint(oracle.make_config(*ck.shape_tuple), ck.shared_weights, seed)   # == the device generator
        _last[name] = (ck, oracle_run(oracle, ck, n, check))
    return _last[name]


@pytest.mark.parametrize("name,env_name", PARAMS)
def test_envelope(l2b, oracle, name, env_name):
    shape, _, n, check, n_prompt, batched, envs = ENVELOPE[name]
    if name in SLOW:
        import psutil
        if psutil.virtual_memory().available < 16 * (1 << 30):
            pytest.skip("needs ~12 GB of free host memory for the payload")
    assert batched_prefill(shape, {}) == batched       # the mirror of pf_prepare agrees with the table
    ck, ref = model(l2b, oracle, name)
    check_context(l2b, ck, n, check, n_prompt, ref, envs[env_name])


# ---- the KV caches at the envelope shapes -------------------------------------------------------------

# pair -> KV format and layout of the context under test, e4m3 scales.  Its twin: a paged context's is the
# contiguous context of the same format, a contiguous bf16 / e4m3 context's the fp32 cache of its rounded
# values (f32-round-bf16 / f32-round-e4m3)
KV_PAIRS = {
    "paged-f32": ("f32", "paged", None),
    "bf16": ("bf16", "contiguous", None),
    "paged-bf16": ("bf16", "paged", None),
    "e4m3-unit": ("e4m3", "contiguous", "unit"),
    "e4m3-stress": ("e4m3", "contiguous", "stress"),
    "paged-e4m3-stress": ("e4m3", "paged", "stress"),
}
LONG = {"ctx4096-h32", "ctx16384-h1"}
# the stress scales cannot give 1 % saturated K and 1 % subnormal V codes here: one row of 4 values
# (seq_len 1), or V rows that repeat (the teacher tokens cycle through a vocabulary of 1 or 3), so the
# smallest |V| is itself the 3 % quantile and stores as 2^-6, not below it
NO_EDGE_FLOOR = {"vocab1", "vocab2-seq1", "ctx1605632"}
KV_PARAMS = [pytest.param(name, env_name, pair, marks=[pytest.mark.slow] if name in SLOW else [],
                          id=f"{name}-{env_name}-{pair}")
             for name, spec in ENVELOPE.items() for env_name in spec[6] for pair in KV_PAIRS
             # 1605632 positions is past the paged layout's limit (test_paged_seq_len_limit)
             if not (name == "ctx1605632" and pair.startswith("paged"))]


def kv_twins(l2b, ck, seed, env, pair):
    """(context under test, its twin, e4m3 scales or None) of KV_PAIRS[pair] on the device-synthesized
    weights of `seed`."""
    from test_gpu_kv_bf16 import kv_pair as bf16_pair
    from test_gpu_kv_e4m3 import kv_pair as e4m3_pair, scales_for
    from test_gpu_kv_paged import twin
    kv, layout, sc = KV_PAIRS[pair]
    scales = scales_for(l2b, ck, sc, seed=seed) if sc else None
    if layout == "paged":
        a, b = twin(l2b, ck, env, kv_format=kv, seed=seed)
        if scales is not None:
            for t in (a, b):
                t.set_kv_scales(scales)
    elif kv == "bf16":
        a, b = bf16_pair(l2b, ck, env, seed=seed)
    else:
        a, b = e4m3_pair(l2b, ck, scales, env, seed=seed)
    return a, b, scales


_cks = {}


def shape_ck(name):
    if name not in _cks:
        from llama2_zig_b200.checkpoint import shape_checkpoint
        _cks.clear()
        _cks[name] = shape_checkpoint(ENVELOPE[name][0])
    return _cks[name]


@pytest.mark.parametrize("name,env_name,pair", KV_PARAMS)
def test_envelope_kv(l2b, name, env_name, pair):
    """Each KV pair bit for bit at each envelope shape and environment: logits at the checked positions,
    the caches below the appended count, forward_argmax, generate_argmax, forward_sample, prefill and
    score; the long shapes fill the cache by prefill up to the checked tail and add a forward_batch and a
    forward_ragged of 4 sessions at different page offsets near the end of the context."""
    from test_gpu_bf16 import _eq
    from test_gpu_kv_e4m3 import STRESS_ROWS, check_edges
    from test_gpu_kv_paged import same_rows
    from test_gpu_transformer import teacher_tokens
    from test_gpu_variants import l2b_env
    shape, seed, n, check, n_prompt, _, envs = ENVELOPE[name]
    S, V = shape[6], abs(shape[5])
    env = envs[env_name]
    ck = shape_ck(name)
    a, b, scales = kv_twins(l2b, ck, seed, env, pair)
    toks = teacher_tokens(n, V)
    with a, b:
        start = check[0] if name in LONG else 0
        if start:
            _eq(a.prefill(toks[:start]), b.prefill(toks[:start]), f"prefill to {start}")
        for pos in range(start, n):
            la, lb = a.forward(toks[pos], pos), b.forward(toks[pos], pos)
            if pos in check:
                _eq(la, lb, f"logits at {pos}")
        same_rows(a, b, n, "forward")
        for pos in check[:3]:
            assert a.forward_argmax(toks[pos], pos) == b.forward_argmax(toks[pos], pos), pos

        if name in LONG:                               # forks of 4 sessions at page offsets 58, 0, 31, 56
            with l2b_env(env):
                sa, sb = [a.session() for _ in range(4)], [b.session() for _ in range(4)]
            try:
                ps = [S - 70, S - 64, S - 33, S - 8]
                for t, ss in ((a, sa), (b, sb)):
                    for s, q in zip(ss, ps):
                        l2b.fork(t, [s], q)
                _eq(l2b.forward_batch(sa, [toks[q] for q in ps], ps),
                    l2b.forward_batch(sb, [toks[q] for q in ps], ps), "forward_batch")
                pos = [q + 1 for q in ps]
                runs = [toks[q:q + k] for q, k in zip(pos, (3, 4, 2, 1))]
                _eq(l2b.forward_ragged(sa, runs, pos), l2b.forward_ragged(sb, runs, pos), "forward_ragged")
                for x, y, q, r in zip(sa, sb, pos, runs):
                    same_rows(x, y, q + len(r), "sessions")
            finally:
                for s in sa + sb:
                    s.close()

        steps = min(16, S)
        gen = teacher_tokens(steps + 1, V)
        forced = np.full(steps, -1, np.int32)
        forced[:steps // 2] = gen[1:steps // 2 + 1]
        for t in (a, b):
            t.reset()
        _eq(a.generate_argmax(gen[0], 0, steps, forced=forced, stop_on_bos=False),
            b.generate_argmax(gen[0], 0, steps, forced=forced, stop_on_bos=False), "generate_argmax")
        for t in (a, b):
            t.reset()
        _eq(a.prefill(toks[:n_prompt]), b.prefill(toks[:n_prompt]), "prefill logits")
        same_rows(a, b, n_prompt, "prefill")
        p = min(n_prompt, n - 1)
        if V > 1:                                      # a 1-entry vocabulary is refused by the sampler
            pa, ca = a.forward_sample(toks[p], p, 0.8, 0.9)
            pb, cb = b.forward_sample(toks[p], p, 0.8, 0.9)
            _eq(pa, pb, "forward_sample probs")
            assert (ca is None) == (cb is None) and (ca is None or np.array_equal(ca, cb))
        for t in (a, b):
            t.reset()
        for x, y, what in zip(a.score(toks[:n_prompt]), b.score(toks[:n_prompt]), ("log-probs", "greedy")):
            _eq(x, y, f"score {what}")

        if KV_PAIRS[pair][2] == "stress" and name not in NO_EDGE_FLOOR:
            m = min(S, STRESS_ROWS)                    # the rows the stress scales were set from
            for t in (a, b):
                t.reset()
            cal = teacher_tokens(m, V)
            _eq(a.prefill(cal), b.prefill(cal), "prefill of the calibration rows")
            same_rows(a, b, m, "prefill of the calibration rows")
            check_edges(a, scales, m, name)


# ---- the paged layout's seq_len limits ---------------------------------------------------------------

# 1-layer models at the paged seq_len limits (the KV pool grows with the rows in use).  tiny: the longest
# paged context create accepts (the 3-pass score buffer and its page staging fill 200 KiB).  hs256 / hs192:
# attn_wo_kernel<8> / <6> (fused by default at dim <= 512), whose page staging of ceil(seq_len / 8)-row
# cluster splits passes the 48 KiB a kernel gets without opting in after 891,384 / 1,448,440 positions;
# 1,556,832 / 1,558,816 are their paged limits
PAGED_LIMITS = {
    "tiny-1556832": (4, 4, 1, 1, 1, -3, 1556832),
    "hs256-891384": (512, 516, 1, 2, 1, -97, 891384),
    "hs256-891385": (512, 516, 1, 2, 1, -97, 891385),
    "hs256-1556832": (512, 516, 1, 2, 1, -97, 1556832),
    "hs192-1448441": (384, 388, 1, 2, 1, -97, 1448441),
    "hs192-1558816": (384, 388, 1, 2, 1, -97, 1558816),
}


def head_rows(t, which, n):
    """Rows [0, n) of layer 0 of the key (4) or value (5) cache of a 1-layer context.  l2b_read_state
    takes a buffer of the whole cache; only the rows are kept."""
    from llama2_zig_b200.binding import FP
    ck = t.ck
    kvd = ck.dim // ck.n_heads * ck.n_kv_heads
    buf = np.empty(ck.n_layers * ck.seq_len * kvd, np.float32)
    got = C.c_uint64()
    assert t.lib.l2b_read_state(t.h, which, buf.ctypes.data_as(FP), buf.size, C.byref(got)) == 0
    assert got.value == buf.size
    return buf[:n * kvd].copy()


def _limit_run(l2b, t, V):
    """A few positions and one forward_batch of t and a session: the outputs and the rows in use."""
    from test_gpu_transformer import teacher_tokens
    toks = teacher_tokens(8, V)
    out = [(f"logits at {p}", t.forward(toks[p], p)) for p in range(5)]
    s = t.session()
    try:
        s.prefill(toks[:2], want_logits=False)
        out.append(("forward_batch", l2b.forward_batch([t, s], [toks[5], toks[2]], [5, 2])))
        for i, (x, n) in enumerate(((t, 6), (s, 3))):
            out += [(f"context {i} {c} rows", head_rows(x, w, n)) for w, c in ((4, "key"), (5, "value"))]
    finally:
        s.close()
    return out


@pytest.mark.parametrize("name", list(PAGED_LIMITS))
def test_paged_seq_len_limit(l2b, name):
    """Paged contexts at the paged seq_len limits create, run and equal their contiguous twins bit for bit.
    The twins are created one at a time: the contiguous one holds up to 3.2 GB of cache."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    from test_gpu_bf16 import _eq
    shape = PAGED_LIMITS[name]
    ck = shape_checkpoint(shape)
    got = {}
    for layout in ("paged", "contiguous"):
        with l2b.Transformer(ck, 69, kv_layout=layout) as t:
            got[layout] = _limit_run(l2b, t, ck.vocab_size)
    for (what, x), (_, y) in zip(got["paged"], got["contiguous"]):
        _eq(x, y, what)


def _create_synthetic(l2b, shape, fmt=0):
    lib = l2b.load_library()
    cfg = l2b.L2BConfig(*shape[:5], abs(shape[5]), shape[6], 1 if shape[5] > 0 else 0)
    h = C.c_void_p()
    if fmt:
        rc = lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt)
    else:
        rc = lib.l2b_create_synthetic(C.byref(h), C.byref(cfg), 1, None)
    msg = lib.l2b_last_error(None).decode()
    if h.value:
        lib.l2b_destroy(h)
    return rc, h.value, msg


@pytest.mark.parametrize("shape,fmt,why", [
    # w2's 57604-float input is past the shared memory of every GEMV kernel (the warm-up step finds it)
    ((1024, 57604, 1, 8, 2, -1000, 64), 0, "activation vector too large for shared memory"),
    # one position more than the 3-pass kernel's score buffer holds per split (32 splits)
    ((4, 4, 1, 1, 1, -3, 1605633), 0, "seq_len too large"),
    # paged: one position more than the score buffer and its split's page staging hold
    ((4, 4, 1, 1, 1, -3, 1556833), 0x800, "seq_len too large"),          # L2B_KV_PAGED
], ids=["x-hid57604", "ctx1605633", "paged-ctx1556833"])
def test_envelope_refused_at_create(l2b, shape, fmt, why):
    """Just past a shared-memory limit l2b_create returns L2B_ERR_UNSUPPORTED (not a CUDA error) with a
    message, and hands back no context."""
    rc, h, msg = _create_synthetic(l2b, shape, fmt)
    assert rc == -2, (rc, msg)
    assert h is None
    assert why in msg, msg
