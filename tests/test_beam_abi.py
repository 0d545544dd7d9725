"""CPU: beam search's entry points and the checks that come before any device is touched.

- L2B_BEAM_MAX is in the header and the binding; l2b_beam_search and l2b_op_logprob_topk are declared,
  exported and typed (test_abi.py checks every declared symbol is exported).
- Every NULL or out-of-range argument of l2b_op_logprob_topk is refused with INVALID_ARG before the device
  is looked for; a valid call on a machine without a device reaches NO_DEVICE.
- l2b_beam_search with a NULL src is refused with INVALID_ARG whatever else it is given (every other
  refusal needs a context, so tests/test_gpu_beam.py checks those).
- The Python wrappers raise L2BError with the status.

What the two calls compute is checked on the GPU (tests/test_gpu_beam.py).
"""
import ctypes as C

import numpy as np
import pytest


def _has_device():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_declared_exported_and_typed(l2b):
    lib = l2b.load_library()
    for name in ("l2b_beam_search", "l2b_op_logprob_topk"):
        assert name in l2b.exported_symbols()
        assert hasattr(lib, name) and getattr(lib, name).argtypes, f"{name} has no argtypes in the binding"
    with open(l2b.binding.header_path()) as f:
        text = f.read()
    assert "#define L2B_BEAM_MAX 8" in text
    assert l2b.BEAM_MAX == 8
    assert "#define L2B_ABI_VERSION 2" in text


def test_logprob_topk_refusals(l2b):
    from llama2_zig_b200.binding import FP, L2BProbIndex
    lib = l2b.load_library()
    x = np.linspace(-3, 3, 40).astype(np.float32)
    xp = x.ctypes.data_as(FP)
    out = (L2BProbIndex * 20)()
    bad = [(None, 40, 4, out), (xp, 40, 4, None), (xp, 0, 1, out), (xp, -3, 1, out), (xp, 40, 0, out),
           (xp, 40, -1, out), (xp, 3, 4, out), (xp, 40, 17, out), (xp, 16, 17, out)]
    for args in bad:
        assert lib.l2b_op_logprob_topk(0, *args) == -1, args
    for k in (1, 16):
        with pytest.raises(l2b.L2BError) as e:
            l2b.logprob_topk(x[:k - 1] if k > 1 else x[:0], k)
        assert e.value.status == -1
    with pytest.raises(l2b.L2BError) as e:
        l2b.logprob_topk(x, 17)
    assert e.value.status == -1
    if _has_device():
        return
    for n, k in ((40, 1), (40, 16), (16, 16)):   # a valid call reaches the device check
        assert lib.l2b_op_logprob_topk(0, xp, n, k, out) == -4


def test_beam_search_null_src(l2b):
    from llama2_zig_b200.binding import FP, IP
    lib = l2b.load_library()
    toks = np.zeros(64, np.int32)
    lens = np.zeros(8, np.int32)
    lps = np.zeros(8, np.float32)
    ran = C.c_int32(7)
    beams = (C.c_void_p * 2)(None, None)
    tp, lp_, fp = toks.ctypes.data_as(IP), lens.ctypes.data_as(IP), lps.ctypes.data_as(FP)
    for args in ((1, 0, beams, 2, 4, 1, tp, lp_, fp, C.byref(ran)),
                 (1, 0, None, 2, 4, 1, tp, lp_, fp, None),
                 (1, 0, beams, 0, 4, 0, None, None, None, None),
                 (-1, -5, beams, 9, -1, 1, tp, lp_, fp, C.byref(ran))):
        assert lib.l2b_beam_search(None, *args) == -1, args
        assert b"src is NULL" in lib.l2b_last_error(None)
    assert ran.value == 7 and not toks.any() and not lens.any() and not lps.any()
    with pytest.raises(l2b.L2BError) as e:
        l2b.beam_search(None, 1, 0, [None, None], 4)
    assert e.value.status == -1
