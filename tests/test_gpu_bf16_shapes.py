"""GPU: bf16 device weights at the shape envelope, on NaN-poisoned sessions, and at full llama2-7B depth.

- Envelope: every shape of test_gpu_envelope.ENVELOPE is accepted in bf16 (the row padding to 8 elements
  keeps every TMA copy legal, including n = 4 mod 8) and its bf16 context, generated on the device,
  equals bitwise an fp32 context of the host payload with its matrices rounded: logits at the checked
  positions and the KV cache.  The shapes fp32 refuses, bf16 refuses with the same status and message.
- Stale rows: test_gpu_stale_rows' paths on a bf16 S and B whose embedding row P is NaN.  NaN survives
  the rounding (the poisoned session's prefill is all NaN), and no path reads or writes KV rows past a
  stream's end (bitwise equal to the clean twin session, every output finite).
- Full depth (slow, ~40 GB of device memory): the llama2-7B synthetic shape, seed 7, in bf16 equals an
  fp32 context of the rounded host payload bitwise at 4 positions and over 32 generate_argmax steps.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_bf16 import _eq, round_matrices
from test_gpu_envelope import ENVELOPE, SLOW
from test_gpu_stale_rows import (checkpoint, path_fork, path_generate, path_generate_batch,  # noqa: F401
                                 path_prefill, path_ragged, path_batch, path_score, path_speculative, path_verify,
                                 poison_token, stream_ends)
from test_gpu_transformer import teacher_tokens
from test_gpu_variants import l2b_env
from test_gpu_verify_sample import host  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def twin_check(l2b, ck, rk, seed, n, check, env):
    """bf16 context of the synthetic seed (device generator) against the fp32 context of rk's payload:
    teacher-forced, positions before check[0] prefilled when the run is long."""
    toks = teacher_tokens(n, ck.vocab_size)
    with l2b_env(env), l2b.Transformer(ck, synthetic_seed=seed, weight_format="bf16") as b, l2b.Transformer(rk) as f:
        start = check[0] if n > 64 else 0
        if start:
            b.prefill(toks[:start], want_logits=False)
            f.prefill(toks[:start], want_logits=False)
        for pos in range(start, n):
            lb, lf = b.forward(toks[pos], pos), f.forward(toks[pos], pos)
            if pos in check:
                _eq(lb, lf, f"logits at {pos}")
        _eq(b.state("key_cache"), f.state("key_cache"), "key cache")
        assert b.weight_info()[1] == int((ck.data != rk.data).sum())


ENV_PARAMS = [pytest.param(name, marks=[pytest.mark.slow] if name in SLOW else [], id=name) for name in ENVELOPE]


@pytest.mark.parametrize("name", ENV_PARAMS)
def test_envelope_bf16(l2b, oracle, name):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    shape, seed, n, check = ENVELOPE[name][:4]
    if name in SLOW:
        import psutil
        if psutil.virtual_memory().available < 24 * (1 << 30):
            pytest.skip("needs ~20 GB of free host memory for the payloads")
    ck = shape_checkpoint(shape)
    ck.data = l2b.synth_checkpoint_host(ck, seed)
    rk = shape_checkpoint(shape, round_matrices(l2b, ck, ck.data))
    twin_check(l2b, ck, rk, seed, n, check, {})


@pytest.mark.parametrize("shape", [(1024, 57604, 1, 8, 2, -1000, 64), (4, 4, 1, 1, 1, -3, 1605633)],
                         ids=["x-hid57604", "ctx1605633"])
def test_envelope_refused_bf16(l2b, shape):
    lib = l2b.load_library()
    cfg = l2b.L2BConfig(*shape[:5], abs(shape[5]), shape[6], 1 if shape[5] > 0 else 0)
    out = []
    for create in (lambda h: lib.l2b_create_synthetic(C.byref(h), C.byref(cfg), 1, None),
                   lambda h: lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, 1)):
        h = C.c_void_p()
        rc = create(h)
        out.append((rc, lib.l2b_last_error(None).decode()))
        assert not h.value
    assert out[0][0] == -2 and out[0] == out[1], out


# ---- stale rows ---------------------------------------------------------------------------------------

STALE_PATHS = {"generate": path_generate, "prefill": path_prefill, "score": path_score, "batch": path_batch,
               "ragged": path_ragged, "verify": path_verify, "generate-batch": path_generate_batch,
               "fork": path_fork, "speculative": None}
_poisoned = {}


@pytest.fixture(scope="module", autouse=True)
def _close_poisoned():
    yield
    for m, _, _ in _poisoned.values():
        m.close()
    _poisoned.clear()


def poisoned_bf16(l2b, oracle, name):
    if name not in _poisoned:
        for m, _, _ in _poisoned.values():
            m.close()
        _poisoned.clear()
        ck = checkpoint(l2b, oracle, name)
        P = poison_token(ck)
        data = ck.data.copy()
        data[P * ck.dim:(P + 1) * ck.dim] = np.nan
        pck = type(ck)(**{**ck.__dict__, "data": data})
        _poisoned[name] = (l2b.Transformer(pck, weight_format="bf16"), ck, P)
    return _poisoned[name]


@pytest.mark.parametrize("path", list(STALE_PATHS))
@pytest.mark.parametrize("name", ["S", "B"])
def test_stale_rows_bf16(l2b, oracle, host, name, path):  # noqa: F811
    m, ck, P = poisoned_bf16(l2b, oracle, name)
    assert m.weight_info()[0] == "bf16"
    ts = stream_ends(ck)
    if path == "speculative":
        path_speculative(l2b, host, m, P, ts)
    else:
        STALE_PATHS[path](l2b, m, P, ts)


# ---- full depth ---------------------------------------------------------------------------------------

@pytest.mark.slow
def test_llama2_7b_bf16_twin(l2b):
    import psutil
    if psutil.virtual_memory().available < 64 * (1 << 30):
        pytest.skip("needs ~60 GB of free host memory for the payloads")
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint("llama2-7B")
    ck.data = l2b.synth_checkpoint_host(ck, 7)
    rk = shape_checkpoint("llama2-7B", round_matrices(l2b, ck, ck.data))
    ck.data = None
    toks = teacher_tokens(8, rk.vocab_size)
    with l2b.Transformer(rk, synthetic_seed=7, weight_format="bf16") as b, l2b.Transformer(rk) as f:
        for pos in range(4):
            _eq(b.forward(toks[pos], pos), f.forward(toks[pos], pos), f"7B logits at {pos}")
        _eq(b.generate_argmax(toks[4], 4, 32, stop_on_bos=False), f.generate_argmax(toks[4], 4, 32, stop_on_bos=False),
            "7B generate_argmax")
        b.reset(); f.reset()
        _eq(b.prefill(toks[:8]), f.prefill(toks[:8]), "7B prefill")
