"""GPU: q8 device weights at the shape envelope, on stale KV rows, and at full llama2-7B depth.

- Envelope: every shape of test_gpu_envelope.ENVELOPE is accepted in q8 (row records padded to 16 bytes
  keep every TMA copy legal, short last groups included) and its q8 context, generated on the device,
  equals bitwise an fp32 context of the host payload with its matrices dequantized: logits at the checked
  positions and the KV cache.  The shapes fp32 refuses, q8 refuses with the same status and message.
- Non-finite weights: a payload with a NaN or inf matrix weight is refused by the q8 upload with
  INVALID_ARG and no context; the same payload still loads as fp32.
- Stale rows: a q8 model cannot hold the NaN embedding row test_gpu_stale_rows poisons with (q8 refuses
  non-finite weights, and every dequantized weight is finite), and the KV cache and the kernels that read
  it are the fp32 ones, which that file checks with NaN.  Here a q8 session whose rows past each stream's
  end hold another stream's values equals a fresh session bitwise on generate, prefill, score, the batch
  calls and the verify call, and the rows those calls may not write keep their bits.
- Full depth (slow, ~35 GB of device memory): the llama2-7B synthetic shape, seed 7, in q8 equals an
  fp32 context of the dequantized host payload bitwise at 4 positions and over 32 generate_argmax steps.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_envelope import ENVELOPE, SLOW
from test_gpu_q8 import _eq
from test_gpu_transformer import teacher_tokens
from test_gpu_variants import l2b_env, payload
from test_q8_abi import dequant_matrices

pytestmark = pytest.mark.gpu


def twin_check(l2b, ck, rk, n_changed, seed, n, check, env):
    """q8 context of the synthetic seed (device generator) against the fp32 context of rk's payload:
    teacher-forced, positions before check[0] prefilled when the run is long."""
    toks = teacher_tokens(n, ck.vocab_size)
    with l2b_env(env), l2b.Transformer(ck, synthetic_seed=seed, weight_format="q8") as b, l2b.Transformer(rk) as f:
        start = check[0] if n > 64 else 0
        if start:
            b.prefill(toks[:start], want_logits=False)
            f.prefill(toks[:start], want_logits=False)
        for pos in range(start, n):
            lb, lf = b.forward(toks[pos], pos), f.forward(toks[pos], pos)
            if pos in check:
                _eq(lb, lf, f"logits at {pos}")
        _eq(b.state("key_cache"), f.state("key_cache"), "key cache")
        assert b.weight_info() == ("q8", n_changed)


ENV_PARAMS = [pytest.param(name, marks=[pytest.mark.slow] if name in SLOW else [], id=name) for name in ENVELOPE]


@pytest.mark.parametrize("name", ENV_PARAMS)
def test_envelope_q8(l2b, name):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    shape, seed, n, check = ENVELOPE[name][:4]
    if name in SLOW:
        import psutil
        if psutil.virtual_memory().available < 24 * (1 << 30):
            pytest.skip("needs ~20 GB of free host memory for the payloads")
    ck = shape_checkpoint(shape)
    ck.data = l2b.synth_checkpoint_host(ck, seed)
    data, n_changed = dequant_matrices(l2b, ck, ck.data)
    rk = shape_checkpoint(shape, data)
    twin_check(l2b, ck, rk, n_changed, seed, n, check, {})


@pytest.mark.parametrize("shape", [(1024, 57604, 1, 8, 2, -1000, 64), (4, 4, 1, 1, 1, -3, 1605633)],
                         ids=["x-hid57604", "ctx1605633"])
def test_envelope_refused_q8(l2b, shape):
    lib = l2b.load_library()
    cfg = l2b.L2BConfig(*shape[:5], abs(shape[5]), shape[6], 1 if shape[5] > 0 else 0)
    out = []
    for create in (lambda h: lib.l2b_create_synthetic(C.byref(h), C.byref(cfg), 1, None),
                   lambda h: lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, 3)):
        h = C.c_void_p()
        rc = create(h)
        out.append((rc, lib.l2b_last_error(None).decode()))
        assert not h.value
    assert out[0][0] == -2 and out[0] == out[1], out


@pytest.mark.parametrize("where", ["embedding", "w2-last", "classifier"])
@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_non_finite_weight_refused(l2b, where, bad):
    from llama2_zig_b200.binding import FP
    from test_q8_abi import matrix_shapes
    ck = payload(l2b, "S")
    data = ck.data.copy()
    shapes = matrix_shapes(ck)
    off = {"embedding": shapes[0][0] + 5, "w2-last": shapes[6][0] + shapes[6][1] * shapes[6][2] - 1,
           "classifier": shapes[-1][0] + 3}[where]
    data[off] = bad
    lib = l2b.load_library()
    cfg = l2b.binding.make_config(ck)
    for _ in range(2):                                   # a refused upload leaves nothing behind
        h = C.c_void_p(12345)
        rc = lib.l2b_create_format(C.byref(h), C.byref(cfg), data.ctypes.data_as(FP), data.size, None, None, 1, 3)
        assert rc == -1 and not h.value
        assert b"non-finite" in lib.l2b_last_error(None)
    bad_ck = type(ck)(**{**ck.__dict__, "data": data})
    with l2b.Transformer(bad_ck) as f:                   # fp32 keeps taking it
        f.forward(1, 0)


# ---- stale rows ---------------------------------------------------------------------------------------

def filled_session(m, ck, toks):
    """A session whose every KV row holds the values of a stream other than `toks`, then reset."""
    s = m.session()
    other = [(t * 7 + 3) % ck.vocab_size for t in toks[:ck.seq_len]]
    s.prefill(other, want_logits=False)
    s.reset()
    return s


@pytest.mark.parametrize("name", ["S", "B"])
def test_stale_rows_q8(l2b, name):
    ck = payload(l2b, name)
    V, T = ck.vocab_size, ck.seq_len
    toks = teacher_tokens(T + 1, V)
    ends = [1, 2, 3, 63, 64, 65, 127, 128, 129, 255, 256, 257, T - 1]
    ends = sorted({e for e in ends if 0 < e < T})
    with l2b.Transformer(ck, weight_format="q8") as m:
        for e in ends:
            a, b = filled_session(m, ck, toks), m.session()
            try:
                before = a.state("key_cache").copy()
                _eq(a.prefill(toks[:e]), b.prefill(toks[:e]), f"prefill to {e}")
                _eq(a.generate_argmax(toks[e], e, min(4, T - e), stop_on_bos=False),
                    b.generate_argmax(toks[e], e, min(4, T - e), stop_on_bos=False), f"generate from {e}")
                n = e + min(4, T - e)
                kv_a, kv_b = a.state("key_cache"), b.state("key_cache")
                rows = kv_a.reshape(ck.n_layers, T, -1)
                _eq(rows[:, :n], kv_b.reshape(ck.n_layers, T, -1)[:, :n], f"appended rows to {n}")
                _eq(rows[:, n:], before.reshape(ck.n_layers, T, -1)[:, n:], f"rows past {n} kept")
                a.reset(); b.reset()
                _eq(a.score(toks[:e + 1])[0], b.score(toks[:e + 1])[0], f"score to {e + 1}")
            finally:
                a.close(); b.close()
        sa = [filled_session(m, ck, toks) for _ in range(4)]
        sb = [m.session() for _ in range(4)]
        try:
            pos = [e for e in ends[:4]]
            for x, y, p in zip(sa, sb, pos):
                x.prefill(toks[:p], want_logits=False)
                y.prefill(toks[:p], want_logits=False)
            t4 = toks[10:14]
            _eq(l2b.forward_batch(sa, t4, pos), l2b.forward_batch(sb, t4, pos), "forward_batch")
            pos = [p + 1 for p in pos]
            runs = [toks[0:1], toks[1:6], toks[6:9], toks[9:11]]
            _eq(l2b.forward_ragged(sa, runs, pos), l2b.forward_ragged(sb, runs, pos), "forward_ragged")
            pos = [p + len(r) for p, r in zip(pos, runs)]
            va = l2b.verify_argmax_ragged(sa, [list(toks[20:24])] * 4, pos)
            vb = l2b.verify_argmax_ragged(sb, [list(toks[20:24])] * 4, pos)
            _eq(va[1], vb[1], "n_accept")
            for x, y in zip(va[0], vb[0]):
                _eq(x, y, "verify tokens")
        finally:
            for s in sa + sb:
                s.close()


# ---- full depth ---------------------------------------------------------------------------------------

@pytest.mark.slow
def test_llama2_7b_q8_twin(l2b):
    import psutil
    if psutil.virtual_memory().available < 64 * (1 << 30):
        pytest.skip("needs ~60 GB of free host memory for the payloads")
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint("llama2-7B")
    ck.data = l2b.synth_checkpoint_host(ck, 7)
    data, _ = dequant_matrices(l2b, ck, ck.data)
    rk = shape_checkpoint("llama2-7B", data)
    ck.data = None
    toks = teacher_tokens(8, rk.vocab_size)
    with l2b.Transformer(rk, synthetic_seed=7, weight_format="q8") as b, l2b.Transformer(rk) as f:
        for pos in range(4):
            _eq(b.forward(toks[pos], pos), f.forward(toks[pos], pos), f"7B logits at {pos}")
        _eq(b.generate_argmax(toks[4], 4, 32, stop_on_bos=False), f.generate_argmax(toks[4], 4, 32, stop_on_bos=False),
            "7B generate_argmax")
        b.reset(); f.reset()
        _eq(b.prefill(toks[:8]), f.prefill(toks[:8]), "7B prefill")
