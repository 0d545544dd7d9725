"""CPU: the paged KV layout's entry points and the checks that come before any device is touched.

- L2B_KV_PAGED and L2B_KV_PAGE_ROWS are in the header and the binding; l2b_kv_pool_info and
  l2b_kv_pool_limit are declared, exported and typed.
- L2B_KV_PAGED is a flag of l2b_create_format / l2b_create_synthetic_format's weight_format: with every
  weight format and KV format it passes the format check, with more than one GPU it is refused
  (UNSUPPORTED), and a valid paged create on a machine without a device reaches NO_DEVICE.
- The pool calls refuse NULL arguments; the Python layer refuses an unknown kv_layout and a multi-GPU
  paged model before it loads anything.

What a paged context computes is checked on the GPU (tests/test_gpu_kv_paged.py).
"""
import ctypes as C

import numpy as np
import pytest

KV_PAGED, PAGE_ROWS = 0x800, 64
FORMATS = [wf | kv | KV_PAGED for wf in (0, 1, 3) for kv in (0, 0x100, 0x200)]


def _has_device():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_declared_exported_and_typed(l2b):
    lib = l2b.load_library()
    for name in ("l2b_kv_pool_info", "l2b_kv_pool_limit"):
        assert name in l2b.exported_symbols()
        assert hasattr(lib, name) and getattr(lib, name).argtypes, f"{name} has no argtypes in the binding"
    with open(l2b.binding.header_path()) as f:
        text = f.read()
    assert "#define L2B_KV_PAGED 0x800" in text and "#define L2B_KV_PAGE_ROWS 64" in text
    assert l2b.KV_PAGED == KV_PAGED and l2b.KV_PAGE_ROWS == PAGE_ROWS
    assert l2b.KV_FORMATS == {"f32": 0, "bf16": 0x100, "f32-round-bf16": 0x200}
    assert l2b.WEIGHT_FORMATS == {"f32": 0, "bf16": 1} and l2b.QUANT_FORMATS == {"q8": 3}


def test_format_checks_come_before_the_device(l2b):
    from llama2_zig_b200.binding import L2BConfig, FP
    lib = l2b.load_library()
    h = C.c_void_p()
    cfg = L2BConfig(288, 768, 6, 6, 6, 32000, 256, 1)
    n = int(lib.l2b_checkpoint_floats(C.byref(cfg)))
    data = np.zeros(n, np.float32)
    dp = data.ctypes.data_as(FP)
    # the paged flag does not make an unknown format known
    for fmt in (KV_PAGED | 0x400, KV_PAGED | 0x300, KV_PAGED | 2, KV_PAGED | 0x10000):
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -1, fmt
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -1, fmt
        assert b"format" in lib.l2b_last_error(None)
    for fmt in FORMATS:
        for g in (2, 4, 8):
            assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, g, fmt) == -2, (fmt, g)
            assert b"single-GPU" in lib.l2b_last_error(None)
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), None, n, None, None, 1, fmt) == -1
        bad = L2BConfig(36, 768, 6, 6, 6, 32000, 256, 1)
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(bad), 1, fmt) == -2
    assert not h.value
    if _has_device():
        return
    for fmt in FORMATS:   # a valid call reaches the device check
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -4
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -4
    assert not h.value


def test_pool_calls_refuse_null(l2b):
    lib = l2b.load_library()
    r, b, u, a = C.c_int32(), C.c_uint64(), C.c_uint64(), C.c_uint64()
    assert lib.l2b_kv_pool_info(None, C.byref(r), C.byref(b), C.byref(u), C.byref(a)) == -1
    assert lib.l2b_kv_pool_limit(None, 0) == -1
    assert lib.l2b_kv_pool_limit(None, 5) == -1


def test_python_refusals(l2b):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint("stories15M")
    with pytest.raises(ValueError, match="kv_layout"):
        l2b.Transformer(ck, synthetic_seed=1, kv_layout="blocked")
    for kw in ({"n_gpus": 2}, {"world_size": 2}, {"device": 1}):
        with pytest.raises(ValueError, match="single-GPU"):
            l2b.Transformer(ck, synthetic_seed=1, kv_layout="paged", **kw)
