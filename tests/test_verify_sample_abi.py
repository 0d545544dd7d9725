"""CPU: l2b_verify_sample_ragged refuses NULL arguments and empty batches before touching CUDA."""
import ctypes as C

import pytest


def test_verify_sample_refuses_null_arguments(l2b):
    lib = l2b.load_library()
    none = (C.c_void_p * 2)()                                           # two NULL sessions
    lens, toks, pos = (C.c_int32 * 2)(2, 1), (C.c_int32 * 3)(1, 2, 3), (C.c_int32 * 2)(0, 0)
    temp, top_p = (C.c_float * 2)(1.0, 1.0), (C.c_float * 2)(0.9, 0.0)
    probs, cand, n_cand = (C.c_float * 3)(), (l2b.binding.L2BProbIndex * 24)(), (C.c_int32 * 3)()
    f = lib.l2b_verify_sample_ragged
    assert f(None, 2, lens, toks, pos, temp, top_p, probs, cand, 8, n_cand) == -1       # NULL sessions
    assert f(none, 2, lens, toks, pos, temp, top_p, probs, cand, 8, n_cand) == -1       # NULL sessions[0]
    assert f(none, 0, lens, toks, pos, temp, top_p, probs, cand, 8, n_cand) == -1       # n < 1
    assert f(none, -1, lens, toks, pos, temp, top_p, probs, cand, 8, n_cand) == -1      # n < 0
    assert f(none, 2, None, None, None, None, None, None, None, 0, None) == -1
    assert b"sessions" in lib.l2b_last_error(None)


def test_verify_sample_without_sessions_raises(l2b):
    with pytest.raises(l2b.L2BError) as e:
        l2b.verify_sample_ragged([], [], [], [], [])
    assert e.value.status == -1


def test_verify_sample_is_declared_and_exported(l2b):
    assert "l2b_verify_sample_ragged" in l2b.exported_symbols()
    assert hasattr(l2b.load_library(), "l2b_verify_sample_ragged")
