"""CPU: l2b_score and l2b_op_logprob refuse missing arguments before touching CUDA."""
import ctypes as C

import numpy as np
import pytest


def test_score_refuses_null_arguments(l2b):
    lib = l2b.load_library()
    toks = (C.c_int32 * 3)(1, 2, 3)
    lp = (C.c_float * 3)()
    greedy = (C.c_int32 * 3)()
    sc = lib.l2b_score
    assert sc(None, toks, 3, 0, lp, greedy) == -1            # NULL ctx
    assert lib.l2b_last_error(None)
    assert sc(None, None, 3, 0, lp, greedy) == -1            # and NULL tokens
    assert sc(None, toks, 3, 0, None, greedy) == -1          # and NULL logprob
    assert sc(None, toks, 0, 0, lp, greedy) == -1            # and n_tokens < 1
    assert sc(None, toks, -2, 0, lp, None) == -1


def test_op_logprob_refuses_null_pointers(l2b):
    lib = l2b.load_library()
    x = (C.c_float * 4)(0.0, 1.0, 2.0, 3.0)
    out = C.c_float()
    op = lib.l2b_op_logprob
    assert op(0, None, 4, 1, C.byref(out)) == -1             # NULL logits
    assert op(0, x, 4, 1, None) == -1                        # NULL logprob
    assert op(0, x, 0, 0, C.byref(out)) == -1                # n < 1
    assert op(0, x, 4, -1, C.byref(out)) == -1               # target outside [0, n)
    assert op(0, x, 4, 4, C.byref(out)) == -1
    with pytest.raises(l2b.L2BError) as e:
        l2b.logprob(np.zeros(0, np.float32), 0)
    assert e.value.status == -1


def test_score_wrapper_refuses_empty_sequence(l2b):
    t = l2b.Transformer.__new__(l2b.Transformer)            # no context: the NULL check comes first
    t.lib, t.h = l2b.load_library(), C.c_void_p()
    with pytest.raises(l2b.L2BError) as e:
        t.score([])
    assert e.value.status == -1
