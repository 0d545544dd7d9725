"""CPU: l2b_create_session and the batched step refuse missing arguments before touching CUDA."""
import ctypes as C


def test_session_and_batch_refuse_null_arguments(l2b):
    from llama2_zig_b200.binding import FP
    lib = l2b.load_library()
    h = C.c_void_p()
    assert lib.l2b_create_session(C.byref(h), None) == -1          # NULL model
    assert not h.value
    assert lib.l2b_create_session(None, None) == -1
    toks = (C.c_int32 * 2)(1, 2)
    pos = (C.c_int32 * 2)(0, 0)
    rows = (FP * 2)()
    nxt = (C.c_int32 * 2)()
    none = (C.c_void_p * 2)()                                      # two NULL sessions
    # NULL sessions, n = 0, and a NULL sessions[0]
    assert lib.l2b_forward_batch(None, 2, toks, pos, rows) == -1
    assert lib.l2b_forward_batch(none, 0, toks, pos, rows) == -1
    assert lib.l2b_forward_batch(none, 2, toks, pos, rows) == -1
    assert lib.l2b_forward_argmax_batch(None, 2, toks, pos, nxt) == -1
    assert lib.l2b_forward_argmax_batch(none, 0, toks, pos, nxt) == -1
    assert lib.l2b_last_error(None)
    for fn in (l2b.forward_batch, l2b.forward_argmax_batch):
        try:
            fn([], [], [])
        except l2b.L2BError as e:
            assert e.status == -1
        else:
            raise AssertionError("an empty batch was accepted")
