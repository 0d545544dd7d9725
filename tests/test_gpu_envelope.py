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


def _create_synthetic(l2b, shape):
    lib = l2b.load_library()
    cfg = l2b.L2BConfig(*shape[:5], abs(shape[5]), shape[6], 1 if shape[5] > 0 else 0)
    h = C.c_void_p()
    rc = lib.l2b_create_synthetic(C.byref(h), C.byref(cfg), 1, None)
    msg = lib.l2b_last_error(None).decode()
    if h.value:
        lib.l2b_destroy(h)
    return rc, h.value, msg


@pytest.mark.parametrize("shape,why", [
    # w2's 57604-float input is past the shared memory of every GEMV kernel (the warm-up step finds it)
    ((1024, 57604, 1, 8, 2, -1000, 64), "activation vector too large for shared memory"),
    # one position more than the 3-pass kernel's score buffer holds per split (32 splits)
    ((4, 4, 1, 1, 1, -3, 1605633), "seq_len too large"),
], ids=["x-hid57604", "ctx1605633"])
def test_envelope_refused_at_create(l2b, shape, why):
    """Just past a shared-memory limit l2b_create returns L2B_ERR_UNSUPPORTED (not a CUDA error) with a
    message, and hands back no context."""
    rc, h, msg = _create_synthetic(l2b, shape)
    assert rc == -2, (rc, msg)
    assert h is None
    assert why in msg, msg
