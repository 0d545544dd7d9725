"""CPU: the ragged calls (l2b_forward_ragged / _argmax_ragged / _sample_ragged) refuse missing arguments
before touching CUDA."""
import ctypes as C


def test_ragged_refuses_null_arguments(l2b):
    lib = l2b.load_library()
    lens = (C.c_int32 * 2)(2, 1)
    toks = (C.c_int32 * 3)(1, 2, 3)
    pos = (C.c_int32 * 2)(0, 0)
    nxt = (C.c_int32 * 2)()
    rows = (C.POINTER(C.c_float) * 2)()
    temp = (C.c_float * 2)(1.0, 0.8)
    top_p = (C.c_float * 2)(0.9, 0.0)
    cand = (l2b.binding.L2BProbIndex * 16)()
    n_cand = (C.c_int32 * 2)()
    none = (C.c_void_p * 2)()                                           # two NULL sessions
    calls = [lambda s, n, ln: lib.l2b_forward_ragged(s, n, ln, toks, pos, rows),
             lambda s, n, ln: lib.l2b_forward_argmax_ragged(s, n, ln, toks, pos, nxt),
             lambda s, n, ln: lib.l2b_forward_sample_ragged(s, n, ln, toks, pos, temp, top_p, None, cand, 8, n_cand)]
    for fn in calls:
        assert fn(None, 2, lens) == -1                                  # NULL sessions
        assert fn(none, 0, lens) == -1                                  # n = 0
        assert fn(none, -3, lens) == -1                                 # n < 0
        assert fn(none, 2, lens) == -1                                  # NULL sessions[0]
        assert fn(none, 2, None) == -1                                  # and NULL n_tokens
        assert fn(None, 2, None) == -1
    assert lib.l2b_forward_ragged(None, 2, lens, None, None, None) == -1
    assert lib.l2b_forward_argmax_ragged(None, 2, None, None, None, None) == -1
    assert lib.l2b_forward_sample_ragged(None, 2, None, None, None, None, None, None, None, 0, None) == -1
    assert lib.l2b_last_error(None)
    for fn, extra in ((l2b.forward_ragged, ()), (l2b.forward_argmax_ragged, ()),
                      (l2b.forward_sample_ragged, ([], []))):
        try:
            fn([], [], [], *extra)
        except l2b.L2BError as e:
            assert e.status == -1
        else:
            raise AssertionError("an empty ragged call was accepted")
