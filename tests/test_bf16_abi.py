"""CPU: the bf16 weight-format entry points, the library's bf16 rounding, and what rounding costs.

- l2b_create_format, l2b_create_synthetic_format, l2b_weight_info and l2b_round_bf16_host are declared,
  exported and typed by the binding.
- l2b_round_bf16_host equals torch's float32 -> bfloat16 -> float32 round trip bitwise (ties, the largest
  finite bf16, overflow to +-inf, subnormals, +-0, +-inf and 1e6 seeded values over the whole exponent
  range); NaN stays NaN.  The device generator and the upload use the same function (l2b_device.cuh:
  bf16_round_bits), so a bf16 context's weights are these values.
- The format checks come before any device is touched.
- The oracle on a rounded stories15M-shaped payload against the unrounded one: where the greedy streams
  part and the largest logit difference (a measurement, recorded in DESIGN.md §4.5j, not a bar).
"""
import ctypes as C

import numpy as np
import pytest

NEW_SYMBOLS = ["l2b_create_format", "l2b_create_synthetic_format", "l2b_weight_info", "l2b_round_bf16_host"]


def _torch_round(x):
    torch = pytest.importorskip("torch")
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).to(torch.float32).numpy()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_declared_exported_and_typed(l2b):
    lib = l2b.load_library()
    names = l2b.exported_symbols()
    for n in NEW_SYMBOLS:
        assert n in names, f"{n} not declared in llama2_b200.h"
        assert getattr(lib, n).argtypes, f"{n} has no argtypes in the binding"
    assert lib.l2b_abi_version() == 2
    assert l2b.WEIGHT_FORMATS == {"f32": 0, "bf16": 1}


def test_round_matches_torch_on_edge_values(l2b):
    u = np.array([
        0x3F808000, 0x3F818000, 0x3F808001, 0x3F817FFF,   # ties to even (down, up) and either side of a tie
        0x7F7F0000, 0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF,   # largest finite bf16; past it -> inf
        0xFF7F8000, 0x7F800000, 0xFF800000,               # -overflow, +-inf
        0x00000000, 0x80000000,                           # +-0
        0x00000001, 0x00008000, 0x00018000, 0x00010000,   # subnormals: rounded, ties to even, not flushed
        0x807FFFFF, 0x007F8000, 0x00008001,
    ], dtype=np.uint32)
    x = u.view(np.float32).copy()
    want = _torch_round(x)
    got = l2b.round_bf16_host(x.copy())
    assert np.array_equal(_bits(got), _bits(want)), (u[_bits(got) != _bits(want)], _bits(got), _bits(want))
    assert np.isinf(got[6]) and np.isinf(got[7]) and got[8] == -np.inf
    assert got[13] == 0.0 and _bits(got)[14] == 0 and _bits(got)[15] == 0x00020000   # 1.5 ulp -> even


def test_round_matches_torch_on_random_values(l2b):
    rng = np.random.default_rng(20261017)
    u = rng.integers(0, 2**32, size=1_000_000, dtype=np.uint64).astype(np.uint32)
    x = u.view(np.float32)
    x = x[~np.isnan(x)].copy()
    assert x.size > 990_000
    got = l2b.round_bf16_host(x.copy())
    assert np.array_equal(_bits(got), _bits(_torch_round(x)))


def test_nan_stays_nan(l2b):
    u = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FFFFFFF, 0xFF80FFFF], dtype=np.uint32)
    got = l2b.round_bf16_host(u.view(np.float32).copy())
    assert np.isnan(got).all()
    assert np.array_equal(_bits(got) & 0x80000000, u & 0x80000000)   # sign kept
    assert not (_bits(got) & 0xFFFF).any()


def test_round_rejects_non_float32(l2b):
    with pytest.raises(TypeError):
        l2b.round_bf16_host(np.zeros(4, np.float64))


def test_rounded_synthetic_weights_are_bf16_exact(l2b):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint("stories15M")
    data = l2b.synth_checkpoint_host(ck, 15)
    once = l2b.round_bf16_host(data.copy())
    twice = l2b.round_bf16_host(once.copy())
    assert np.array_equal(_bits(once), _bits(twice))
    assert not (_bits(once) & 0xFFFF).any()
    assert (once != data).sum() > data.size // 2        # synthetic weights are not bf16-exact


def test_format_checks_come_before_the_device(l2b):
    from llama2_zig_b200.binding import L2BConfig, FP
    lib = l2b.load_library()
    h = C.c_void_p()
    cfg = L2BConfig(288, 768, 6, 6, 6, 32000, 256, 1)
    n = int(lib.l2b_checkpoint_floats(C.byref(cfg)))
    data = np.zeros(n, np.float32)
    dp = data.ctypes.data_as(FP)
    for fmt in (2, -1, 7):                                 # unknown format
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -1
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -1
        assert b"format" in lib.l2b_last_error(None)
    assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 2, 1) == -2   # bf16 is single-GPU
    assert b"single-GPU" in lib.l2b_last_error(None)
    assert lib.l2b_create_format(C.byref(h), C.byref(cfg), None, n, None, None, 1, 1) == -1  # l2b_create's checks
    assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, 8, None, None, 1, 1) == -1
    bad = L2BConfig(36, 768, 6, 6, 6, 32000, 256, 1)
    assert lib.l2b_create_format(C.byref(h), C.byref(bad), dp, n, None, None, 1, 1) == -2
    assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(bad), 1, 1) == -2
    assert not h.value
    if _has_device():
        return
    for fmt in (0, 1):                                     # a valid call reaches the device check
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -4
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -4
    assert lib.l2b_weight_info(None, None, None) == -1


def _has_device():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_oracle_rounding_cost_stories15m(oracle, l2b):
    """Greedy streams of the oracle on the stories15M-shaped fixture payload, unrounded and rounded:
    the first step where they part and the largest |logit| difference over the teacher-forced run."""
    cfg = oracle.make_config(*oracle.STORIES15M_SHAPE)
    shared = True
    data = oracle.synth_checkpoint(cfg, shared, oracle.STORIES15M_SEED)
    rounded = l2b.round_bf16_host(data.copy())
    a = oracle.OracleModel(cfg, data, shared, W=8, kind="strict")
    b = oracle.OracleModel(cfg, rounded, shared, W=8, kind="strict")
    steps = cfg.seq_len
    _, ga, _ = a.generate(1, steps, stop_on_bos=False)
    _, gb, _ = b.generate(1, steps, stop_on_bos=False)
    differ = np.nonzero(ga != gb)[0]
    first = int(differ[0]) if differ.size else None
    a.close(); b.close()
    a = oracle.OracleModel(cfg, data, shared, W=8, kind="strict")
    b = oracle.OracleModel(cfg, rounded, shared, W=8, kind="strict")
    worst = 0.0
    tok = 1
    for pos in range(steps):
        la, lb = a.forward(tok, pos), b.forward(tok, pos)
        worst = max(worst, float(np.max(np.abs(la - lb)) / np.max(np.abs(la))))
        tok = int(ga[pos])
    print(f"\nbf16 rounding on stories15M-shaped seed {oracle.STORIES15M_SEED}: greedy streams part at step "
          f"{first} of {steps}; max relative logit difference {worst:.3e}")
    assert 0.0 < worst < 0.5
