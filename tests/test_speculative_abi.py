"""CPU: l2b_verify_argmax_ragged and l2b_generate_speculative refuse NULL arguments before touching CUDA."""
import ctypes as C

import pytest


def test_verify_refuses_null_arguments(l2b):
    lib = l2b.load_library()
    none = (C.c_void_p * 2)()                                           # two NULL sessions
    lens, toks, pos = (C.c_int32 * 2)(2, 1), (C.c_int32 * 3)(1, 2, 3), (C.c_int32 * 2)(0, 0)
    greedy, acc = (C.c_int32 * 3)(), (C.c_int32 * 2)()
    assert lib.l2b_verify_argmax_ragged(None, 2, lens, toks, pos, 0, greedy, acc) == -1   # NULL sessions
    assert lib.l2b_verify_argmax_ragged(none, 2, lens, toks, pos, 1, greedy, acc) == -1   # NULL sessions[0]
    assert lib.l2b_verify_argmax_ragged(none, 0, lens, toks, pos, 0, greedy, acc) == -1   # n < 1
    assert lib.l2b_verify_argmax_ragged(none, 2, None, None, None, 0, None, None) == -1
    assert b"sessions" in lib.l2b_last_error(None)


def test_speculative_refuses_null_arguments(l2b):
    lib = l2b.load_library()
    out, done, rounds = (C.c_int32 * 4)(), C.c_int32(), C.c_int32()
    assert lib.l2b_generate_speculative(None, None, 1, 0, 4, 3, 1, out, C.byref(done), C.byref(rounds)) == -1
    assert lib.l2b_generate_speculative(None, None, 1, 0, 4, 3, 1, None, None, None) == -1
    assert b"target" in lib.l2b_last_error(None)


@pytest.mark.parametrize("target", [None, "unopened"])
def test_speculative_without_a_context_raises(l2b, target):
    if target == "unopened":                                            # a handle that holds no context
        target = l2b.Transformer.__new__(l2b.Transformer)
        target.lib = l2b.load_library()
        target.h = C.c_void_p()
        target.ck = None
        with pytest.raises(l2b.L2BError) as e:
            target.generate_speculative(None, 1, 0, 4, 3)
        assert e.value.status == -1
    else:
        with pytest.raises(l2b.L2BError) as e:
            l2b.verify_argmax_ragged([], [], [])
        assert e.value.status == -1
