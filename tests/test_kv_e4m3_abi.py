"""CPU: the fp8 (e4m3) KV-cache format's entry points, its rounding, and the checks that come before any device
is touched.

- L2B_KV_E4M3, L2B_KV_ROUND_E4M3 (its fp32 reference), l2b_kv_scales and l2b_round_e4m3_host are declared,
  exported and typed; the binding's KV_E4M3, KV_ROUND_E4M3 and KV_E4M3_FORMATS are the header's values, and
  KV_FORMATS is unchanged.
- Each flag passes the format check with every weight format, with or without L2B_KV_PAGED; any two of the
  four KV element flags together are an unknown format (INVALID_ARG); more than one GPU is refused
  (UNSUPPORTED); all before any device is touched.
- l2b_round_e4m3_host equals torch.float8_e4m3fn's round trip bit for bit wherever torch rounds to nearest
  even (|v| <= 464), exhaustively over 2^-12 <= |v| < 2^9, and saturates to +-448 beyond, where torch gives
  NaN.  A non-unit scale is fl(e4m3(fl(v / s)) * s) computed in numpy float32.
- The Python layer refuses a multi-GPU e4m3 cache before it loads anything.

What an e4m3-KV context computes is checked on the GPU (tests/test_gpu_kv_e4m3.py).
"""
import ctypes as C

import numpy as np
import pytest
import torch

KV_E4M3, KV_ROUND_E4M3 = 0x1000, 0x2000
ELEM_FLAGS = (0x100, 0x200, KV_E4M3, KV_ROUND_E4M3)
FORMATS = [wf | kv | pg for wf in (0, 1, 3) for kv in (KV_E4M3, KV_ROUND_E4M3) for pg in (0, 0x800)]


def _has_device():
    try:
        return torch.cuda.is_available()
    except Exception:
        return False


def torch_e4m3(v):
    """fl(e4m3(v)) by torch (nearest even; NaN past 464)."""
    return torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(torch.float8_e4m3fn).to(torch.float32).numpy()


def want_e4m3(v, s=np.float32(1.0)):
    """The header's rule restated in numpy float32: u = fl(v / s), saturated to +-448 (inf included, NaN
    kept), rounded by torch, times s."""
    with np.errstate(all="ignore"):
        u = (np.asarray(v, np.float32) / np.float32(s)).astype(np.float32)
        return (torch_e4m3(np.clip(u, -448.0, 448.0)) * np.float32(s)).astype(np.float32)


def same_bits(got, want, what):
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    assert np.array_equal(np.signbit(got[nan]), np.signbit(want[nan])), what
    bad = np.nonzero(got[~nan].view(np.uint32) != want[~nan].view(np.uint32))[0]
    assert bad.size == 0, (what, got[~nan][bad[:5]], want[~nan][bad[:5]])


def test_declared_exported_and_typed(l2b):
    lib = l2b.load_library()
    for name in ("l2b_kv_scales", "l2b_round_e4m3_host"):
        assert name in l2b.exported_symbols()
        assert getattr(lib, name).argtypes, f"{name} has no argtypes in the binding"
    assert lib.l2b_abi_version() == 2
    with open(l2b.binding.header_path()) as f:
        text = f.read()
    assert "#define L2B_KV_E4M3 0x1000" in text and "#define L2B_KV_ROUND_E4M3 0x2000" in text
    assert l2b.KV_E4M3 == KV_E4M3 and l2b.KV_ROUND_E4M3 == KV_ROUND_E4M3
    assert l2b.KV_E4M3_FORMATS == {"e4m3": KV_E4M3, "f32-round-e4m3": KV_ROUND_E4M3}
    assert l2b.KV_FORMATS == {"f32": 0, "bf16": 0x100, "f32-round-bf16": 0x200}


def test_format_checks_come_before_the_device(l2b):
    from llama2_zig_b200.binding import L2BConfig, FP
    lib = l2b.load_library()
    h = C.c_void_p()
    cfg = L2BConfig(288, 768, 6, 6, 6, 32000, 256, 1)
    n = int(lib.l2b_checkpoint_floats(C.byref(cfg)))
    data = np.zeros(n, np.float32)
    dp = data.ctypes.data_as(FP)
    pairs = [a | b for i, a in enumerate(ELEM_FLAGS) for b in ELEM_FLAGS[i + 1:]]
    for fmt in pairs + [p | 0x800 for p in pairs] + [KV_E4M3 | 0x400, KV_E4M3 | 0x10000, KV_ROUND_E4M3 | 2]:
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -1, hex(fmt)
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -1, hex(fmt)
        assert b"format" in lib.l2b_last_error(None)
    for fmt in FORMATS:
        for g in (2, 4, 8):
            assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, g, fmt) == -2, (hex(fmt), g)
            assert b"single-GPU" in lib.l2b_last_error(None)
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), None, n, None, None, 1, fmt) == -1
        bad = L2BConfig(36, 768, 6, 6, 6, 32000, 256, 1)
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(bad), 1, fmt) == -2
    assert not h.value
    ones = np.ones(12, np.float32)
    assert lib.l2b_kv_scales(None, ones.ctypes.data_as(FP), 12) == -1
    assert lib.l2b_kv_scales(None, None, 12) == -1
    if _has_device():
        return
    for fmt in FORMATS:   # a valid call reaches the device check
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -4, hex(fmt)
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -4, hex(fmt)
    assert not h.value


def test_round_exhaustive_against_torch(l2b):
    """Every fp32 bit pattern of both signs with 2^-12 <= |v| < 2^9, one exponent at a time."""
    mant = np.arange(1 << 23, dtype=np.uint32)
    for e in range(127 - 12, 127 + 9):
        bits = np.concatenate([(e << 23) | mant, 0x80000000 | (e << 23) | mant])
        v = bits.view(np.float32)
        got = l2b.round_e4m3_host(v.copy())
        inside = np.abs(v) <= 464.0
        same_bits(got[inside], torch_e4m3(v[inside]), f"exponent {e - 127}")
        assert np.array_equal(got[~inside], np.copysign(np.float32(448.0), v[~inside])), f"exponent {e - 127}"


def test_round_sampled_rest(l2b):
    """A random sample of the other fp32 patterns with |v| <= 464 (below 2^-12: zeros and the smallest codes)."""
    rng = np.random.default_rng(7)
    bits = rng.integers(0, 1 << 32, size=1 << 22, dtype=np.uint64).astype(np.uint32)
    v = bits.view(np.float32)
    v = v[np.abs(v) <= 464.0]
    assert v.size > 1 << 20
    same_bits(l2b.round_e4m3_host(v.copy()), torch_e4m3(v), "sample")


def test_round_named_cases(l2b):
    f = np.float32
    cases = {
        464.0: 448.0,                     # the midpoint of 448 and (the absent) 480: a tie to even
        -464.0: -448.0,
        470.0: 448.0, 1e9: 448.0, np.inf: 448.0, -np.inf: -448.0, -3e38: -448.0,   # saturation (satfinite)
        448.0: 448.0, 447.0: 448.0, 432.0: 448.0, 400.0: 384.0, 424.0: 416.0,      # ties to even near the top
        2.0 ** -10: 0.0, 3 * 2.0 ** -10: 2.0 ** -8, 5 * 2.0 ** -10: 2.0 ** -8,      # subnormal ties
        7.5 * 2.0 ** -9: 2.0 ** -6,       # the last subnormal tie rounds up to the smallest normal
        2.0 ** -9: 2.0 ** -9, 1e-30: 0.0, 1.0: 1.0, 1.0625: 1.0, 1.1875: 1.25, 17.0: 16.0, 18.0: 18.0,
    }
    v = np.array(list(cases), f)
    same_bits(l2b.round_e4m3_host(v.copy()), np.array(list(cases.values()), f), "named cases")
    for x in (470.0, 1e9, np.inf):       # torch has no satfinite rule: NaN there
        assert np.isnan(torch_e4m3(np.array([x], f)))[0]
    z = l2b.round_e4m3_host(np.array([-0.0, 0.0, -1e-30, np.nan, -np.nan], f))
    assert z[0] == 0 and np.signbit(z[0]) and not np.signbit(z[1]) and np.signbit(z[2])
    assert np.isnan(z[3]) and not np.signbit(z[3]) and np.isnan(z[4]) and np.signbit(z[4])


def test_unit_scale_is_identity_on_codes(l2b):
    codes = np.arange(256, dtype=np.uint8)
    vals = torch.from_numpy(codes).view(torch.float8_e4m3fn).to(torch.float32).numpy()
    same_bits(l2b.round_e4m3_host(vals.copy()), vals, "every e4m3 value")


@pytest.mark.parametrize("s", [0.25, 0.0131, 3.7, 1.0 / 448, 2.0 ** -100, 1e30])
def test_scaled_rounding(l2b, s):
    rng = np.random.default_rng(11)
    v = np.concatenate([rng.standard_normal(1 << 16).astype(np.float32) * np.float32(s) * f
                        for f in (1e-4, 0.05, 1, 30, 600)] + [np.array([0, -0.0, np.inf, -np.inf, np.nan], np.float32)])
    same_bits(l2b.round_e4m3_host(v.copy(), s), want_e4m3(v, s), f"scale {s}")


def test_python_refusals(l2b):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint("stories15M")
    for kv in ("e4m3", "f32-round-e4m3"):
        for kw in ({"n_gpus": 2}, {"world_size": 2}, {"device": 1}):
            with pytest.raises(ValueError, match="single-GPU"):
                l2b.Transformer(ck, synthetic_seed=1, kv_format=kv, **kw)
    with pytest.raises(ValueError, match="kv_format"):
        l2b.Transformer(ck, synthetic_seed=1, kv_format="fp8")
    with pytest.raises(TypeError):
        l2b.round_e4m3_host(np.zeros(4, np.float64))
