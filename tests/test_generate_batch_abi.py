"""CPU: l2b_generate_argmax_batch refuses missing arguments before touching CUDA."""
import ctypes as C


def test_generate_batch_refuses_null_arguments(l2b):
    lib = l2b.load_library()
    toks = (C.c_int32 * 2)(1, 2)
    pos = (C.c_int32 * 2)(0, 0)
    out = (C.c_int32 * 8)()
    done = (C.c_int32 * 2)()
    none = (C.c_void_p * 2)()                                      # two NULL sessions
    gen = lib.l2b_generate_argmax_batch
    assert gen(None, 2, toks, pos, 4, None, 1, out, done) == -1    # NULL sessions
    assert gen(none, 0, toks, pos, 4, None, 1, out, done) == -1    # n = 0
    assert gen(none, -3, toks, pos, 4, None, 1, out, done) == -1   # n < 0
    assert gen(none, 2, toks, pos, 4, None, 1, out, done) == -1    # NULL sessions[0]
    assert gen(none, 2, toks, pos, 4, None, 1, None, done) == -1   # and NULL out_next
    assert gen(none, 2, toks, pos, 4, None, 1, out, None) == -1    # and NULL n_done
    assert lib.l2b_last_error(None)
    try:
        l2b.generate_argmax_batch([], [], [], 4)
    except l2b.L2BError as e:
        assert e.status == -1
    else:
        raise AssertionError("an empty batch was accepted")
