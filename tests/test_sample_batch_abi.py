"""CPU: l2b_forward_sample_batch refuses missing arguments before touching CUDA."""
import ctypes as C


def test_sample_batch_refuses_null_arguments(l2b):
    lib = l2b.load_library()
    toks = (C.c_int32 * 2)(1, 2)
    pos = (C.c_int32 * 2)(0, 0)
    temp = (C.c_float * 2)(1.0, 0.8)
    top_p = (C.c_float * 2)(0.9, 0.0)
    cand = (l2b.binding.L2BProbIndex * 16)()
    n_cand = (C.c_int32 * 2)()
    none = (C.c_void_p * 2)()                                                 # two NULL sessions
    fs = lib.l2b_forward_sample_batch
    assert fs(None, 2, toks, pos, temp, top_p, None, cand, 8, n_cand) == -1   # NULL sessions
    assert fs(none, 0, toks, pos, temp, top_p, None, cand, 8, n_cand) == -1   # n = 0
    assert fs(none, -3, toks, pos, temp, top_p, None, cand, 8, n_cand) == -1  # n < 0
    assert fs(none, 2, toks, pos, temp, top_p, None, cand, 8, n_cand) == -1   # NULL sessions[0]
    assert fs(none, 2, toks, pos, None, top_p, None, cand, 8, n_cand) == -1   # and NULL temperature
    assert fs(none, 2, toks, pos, temp, None, None, cand, 8, n_cand) == -1    # and NULL top_p
    assert fs(None, 2, toks, pos, None, None, None, None, 0, None) == -1      # all of them NULL
    assert lib.l2b_last_error(None)
    try:
        l2b.forward_sample_batch([], [], [], [], [])
    except l2b.L2BError as e:
        assert e.status == -1
    else:
        raise AssertionError("an empty batch was accepted")
