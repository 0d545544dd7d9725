"""CPU: l2b_fork refuses a NULL source, a NULL destination array and n_dst < 1 before touching CUDA."""
import ctypes as C

import pytest


def test_fork_refuses_null_arguments(l2b):
    lib = l2b.load_library()
    none = (C.c_void_p * 2)()                                           # two NULL sessions
    assert lib.l2b_fork(None, 0, none, 2) == -1                         # NULL src
    assert lib.l2b_fork(None, 3, None, 2) == -1
    assert lib.l2b_fork(None, 0, none, 0) == -1
    assert lib.l2b_fork(None, -1, none, -5) == -1
    assert b"src" in lib.l2b_last_error(None)


@pytest.mark.parametrize("src", [None, "unopened"])
def test_fork_of_no_destinations_raises(l2b, src):
    if src == "unopened":                                               # a handle that holds no context
        src = l2b.Transformer.__new__(l2b.Transformer)
        src.h = C.c_void_p()
    with pytest.raises(l2b.L2BError) as e:
        l2b.fork(src, [], 0)
    assert e.value.status == -1
