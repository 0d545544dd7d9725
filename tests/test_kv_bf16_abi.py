"""CPU: the bf16 KV-cache format's entry points and the checks that come before any device is touched.

- L2B_KV_BF16, L2B_KV_ROUND_BF16 (its fp32 reference) and l2b_kv_info are declared, exported and typed by
  the binding; the binding's KV_BF16, KV_ROUND_BF16 and KV_FORMATS are the header's values.
- Each is a flag of l2b_create_format / l2b_create_synthetic_format's weight_format: with every weight format
  it passes the format check, both together or any other bit is an unknown format (INVALID_ARG), and with
  more than one GPU it is refused (UNSUPPORTED), all before any device is touched.
- The Python layer refuses an unknown kv_format and a multi-GPU bf16 cache before it loads anything.

What a bf16-KV context computes is checked on the GPU (tests/test_gpu_kv_bf16.py).
"""
import ctypes as C

import numpy as np
import pytest

KV_BF16, KV_ROUND = 0x100, 0x200


def _has_device():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_declared_exported_and_typed(l2b):
    lib = l2b.load_library()
    assert "l2b_kv_info" in l2b.exported_symbols()
    assert lib.l2b_kv_info.argtypes, "l2b_kv_info has no argtypes in the binding"
    assert lib.l2b_abi_version() == 2
    with open(l2b.binding.header_path()) as f:
        text = f.read()
    assert "#define L2B_KV_BF16 0x100" in text and "#define L2B_KV_ROUND_BF16 0x200" in text
    assert l2b.KV_BF16 == KV_BF16 and l2b.KV_ROUND_BF16 == KV_ROUND
    assert l2b.KV_FORMATS == {"f32": 0, "bf16": KV_BF16, "f32-round-bf16": KV_ROUND}
    assert l2b.WEIGHT_FORMATS == {"f32": 0, "bf16": 1} and l2b.QUANT_FORMATS == {"q8": 3}


def test_format_checks_come_before_the_device(l2b):
    from llama2_zig_b200.binding import L2BConfig, FP
    lib = l2b.load_library()
    h = C.c_void_p()
    cfg = L2BConfig(288, 768, 6, 6, 6, 32000, 256, 1)
    n = int(lib.l2b_checkpoint_floats(C.byref(cfg)))
    data = np.zeros(n, np.float32)
    dp = data.ctypes.data_as(FP)
    # unknown bits beside the flags, both flags, and unknown weight formats under them
    for fmt in (0x400, 0x80, KV_BF16 | KV_ROUND, KV_BF16 | 0x400, KV_BF16 | 2, KV_BF16 | 4, KV_ROUND | 7,
                0x10000 | KV_BF16, -1):
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -1, fmt
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -1, fmt
        assert b"format" in lib.l2b_last_error(None)
    for fmt in [wf | kv for wf in (0, 1, 3) for kv in (KV_BF16, KV_ROUND)]:   # single-GPU, any weight format
        for g in (2, 4, 8):
            assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, g, fmt) == -2
            assert b"single-GPU" in lib.l2b_last_error(None)
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), None, n, None, None, 1, fmt) == -1   # l2b_create's checks
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, 8, None, None, 1, fmt) == -1
        bad = L2BConfig(36, 768, 6, 6, 6, 32000, 256, 1)
        assert lib.l2b_create_format(C.byref(h), C.byref(bad), dp, n, None, None, 1, fmt) == -2
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(bad), 1, fmt) == -2
    assert not h.value
    assert lib.l2b_kv_info(None, None, None) == -1
    if _has_device():
        return
    for fmt in [wf | kv for wf in (0, 1, 3) for kv in (KV_BF16, KV_ROUND)]:   # a valid call reaches the device check
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -4
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -4
    assert not h.value


def test_python_refusals(l2b):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint("stories15M")
    with pytest.raises(ValueError, match="kv_format"):
        l2b.Transformer(ck, synthetic_seed=1, kv_format="fp8")
    for kw in ({"n_gpus": 2}, {"world_size": 2}, {"device": 1}):
        with pytest.raises(ValueError, match="single-GPU"):
            l2b.Transformer(ck, synthetic_seed=1, kv_format="bf16", **kw)

