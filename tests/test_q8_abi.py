"""CPU: the q8 weight format's entry points, the library's quantizer, and what quantization costs.

- L2B_WEIGHTS_Q8 and l2b_round_q8_host are declared, exported and typed by the binding (with the
  format entry points bf16 introduced).
- l2b_round_q8_host equals a numpy restatement of the quantizer (include/llama2_b200.h, "device weight
  format") bit for bit, in every dequantized weight and in the count of changed weights: random normal
  rows and the edge rows (an all-zero group, short last groups, values at +-a, ties of w / s, subnormal
  groups, a scale that underflows to 0, a single outlier).  The device generator and the upload use
  the same functions (l2b_device.cuh: q8_scale, q8_code, q8_dequant), so a q8 context's weights are
  these values.
- Every dequantized weight with a normal scale lies within 0.5 * s plus 2 ulps of the weight.
- A non-finite value is refused and leaves the buffer untouched.
- The format checks come before any device is touched.
- The oracle on the dequantized stories15M-shaped payload against the original one: where the greedy
  streams part and the largest logit difference (a measurement, recorded in DESIGN.md §4.5k, not a bar).
"""
import ctypes as C

import numpy as np
import pytest

NEW_SYMBOLS = ["l2b_create_format", "l2b_create_synthetic_format", "l2b_weight_info", "l2b_round_bf16_host",
               "l2b_round_q8_host"]
GROUP = 64


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def q8_numpy(w):
    """The quantizer restated: (dequantized weights, scales [rows][groups]) of a 2-D float32 array."""
    w = np.ascontiguousarray(w, np.float32)
    out = np.empty_like(w)
    scales = []
    for g0 in range(0, w.shape[1], GROUP):
        blk = w[:, g0:g0 + GROUP]
        a = np.max(np.abs(blk), axis=1, keepdims=True)
        s = a / np.float32(127.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            t = np.rint(blk / s)
        q = np.where(np.isnan(t), np.float32(0), np.clip(t, -127, 127))
        q = np.where(a == 0, np.float32(0), q).astype(np.int8)
        out[:, g0:g0 + GROUP] = q.astype(np.float32) * s
        scales.append(s[:, 0])
    return out, np.stack(scales, axis=1)


def matrix_shapes(ck):
    """(offset, rows, cols) of each matrix tensor of a payload in checkpoint order (a stacked
    [L][rows][cols] tensor is L * rows rows): what a q8 context quantizes.  Gains and RoPE stay fp32."""
    d, h, L, V = ck.dim, ck.hidden_dim, ck.n_layers, ck.vocab_size
    kvd = d // ck.n_heads * ck.n_kv_heads
    hs = d // ck.n_heads
    parts = [(V, d), ("g", L * d), (L * d, d), (L * kvd, d), (L * kvd, d), (L * d, d), ("g", L * d),
             (L * h, d), (L * d, h), (L * h, d), ("g", d), ("g", ck.seq_len * hs)]
    if not ck.shared_weights:
        parts.append((V, d))
    out, off = [], 0
    for rows, n in parts:
        if rows == "g":
            off += n
        else:
            out.append((off, rows, n))
            off += rows * n
    return out


def dequant_matrices(l2b, ck, data):
    """(dq(P), count): the payload with every matrix weight replaced by its q8 dequantized value."""
    data = data.copy()
    changed = 0
    for off, rows, cols in matrix_shapes(ck):
        seg = np.ascontiguousarray(data[off:off + rows * cols]).reshape(rows, cols)
        changed += l2b.round_q8_host(seg)
        data[off:off + rows * cols] = seg.ravel()
    return data, changed


def _check_rows(l2b, w):
    want, scales = q8_numpy(w)
    got = w.copy()
    n = l2b.round_q8_host(got)
    assert np.array_equal(_bits(got), _bits(want)), int((_bits(got) != _bits(want)).sum())
    assert n == int((_bits(want) != _bits(w)).sum())
    # the error bound, where the group's scale is a normal number
    s = np.repeat(scales, GROUP, axis=1)[:, :w.shape[1]].astype(np.float64)
    normal = s >= np.finfo(np.float32).tiny
    err = np.abs(got.astype(np.float64) - w.astype(np.float64))
    bound = 0.5 * s + 2 * np.spacing(np.abs(w)).astype(np.float64)
    assert (err[normal] <= bound[normal]).all()
    return got, n


def test_declared_exported_and_typed(l2b):
    lib = l2b.load_library()
    names = l2b.exported_symbols()
    for n in NEW_SYMBOLS:
        assert n in names, f"{n} not declared in llama2_b200.h"
        assert getattr(lib, n).argtypes, f"{n} has no argtypes in the binding"
    assert lib.l2b_abi_version() == 2
    assert l2b.WEIGHT_FORMATS == {"f32": 0, "bf16": 1} and l2b.QUANT_FORMATS == {"q8": 3}
    assert l2b.Q8_GROUP == GROUP
    with open(l2b.binding.header_path()) as f:
        text = f.read()
    assert "L2B_WEIGHTS_Q8 = 3" in text and "#define L2B_Q8_GROUP 64" in text


@pytest.mark.parametrize("cols", [4, 60, 64, 772, 4096, 11008])
def test_round_matches_numpy_on_random_rows(l2b, cols):
    rng = np.random.default_rng(cols)
    w = (rng.standard_normal((24, cols)) * 0.02).astype(np.float32)
    _, n = _check_rows(l2b, w)
    assert n > w.size // 2


def test_round_matches_numpy_on_edge_rows(l2b):
    sub = np.float32(1.4e-45)                                   # the smallest subnormal
    rows = []
    r = np.linspace(-1, 1, 772).astype(np.float32)
    r[64:128] = 0.0                                             # an all-zero group
    r[128:192] = -0.0
    rows.append(r)
    r = np.zeros(772, np.float32)                               # ties of w / s: a = 127 gives s = 1
    r[0:64] = np.arange(64, dtype=np.float32) - np.float32(31.5)
    r[0] = 127.0
    r[64:128] = np.float32(0.5) * (np.arange(64, dtype=np.float32) - 32)
    r[64] = -127.0
    r[768:772] = [127.0, 2.5, -3.5, 0.5]                        # the short last group (4 of 772)
    rows.append(r)
    r = np.full(772, 0.01, np.float32)                          # values at exactly +-a
    r[0:64:2] = -0.25
    r[1:64:2] = 0.25
    r[64:128] = 3.0e38
    r[128:192] = -3.0e38
    r[192] = 100.0                                              # a single outlier sets the group's scale
    rows.append(r)
    r = np.zeros(772, np.float32)                               # subnormal groups
    r[0:64] = np.arange(64, dtype=np.float32) * sub * 7
    r[64:128] = -np.arange(64, dtype=np.float32) * sub
    r[128:192] = sub * 190                                      # s = 1 subnormal step: the clamp at 127
    r[129] = sub * 3
    r[192:256] = sub * 3                                        # s underflows to 0: q = +-127 or 0
    r[193] = 0.0
    r[194] = -sub
    r[256:320] = np.float32(1.0e-39)
    rows.append(r)
    w = np.stack(rows)
    got, _ = _check_rows(l2b, w)
    assert (got[0, 64:192] == 0).all()
    assert np.array_equal(got[1, 1:64], np.rint(w[1, 1:64])) and np.array_equal(got[1, 65:128], np.rint(w[1, 65:128]))
    assert list(got[1, 768:772]) == [127.0, 2.0, -4.0, 0.0]   # rint to nearest even
    assert got[2, 64] == np.float32(3.0e38) and got[2, 128] == np.float32(-3.0e38)
    assert got[2, 0] == -0.25 and got[2, 1] == 0.25
    assert (_bits(got[3, 192:256]) & 0x7FFFFFFF == 0).all()
    short = np.array([[0.1, -0.2, 0.3, 0.04]], np.float32)   # n = 4: one short group
    _check_rows(l2b, short)


def test_round_is_idempotent_on_synthetic_payload(l2b):
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint("stories15M")
    data = l2b.synth_checkpoint_host(ck, 15)
    once, n1 = dequant_matrices(l2b, ck, data)
    twice, n2 = dequant_matrices(l2b, ck, once)
    assert n1 > data.size // 2 and n2 == 0                     # synthetic weights are not q8-exact
    assert np.array_equal(_bits(once), _bits(twice))
    off, rows, cols = matrix_shapes(ck)[2]                     # wq, against the numpy restatement
    want, _ = q8_numpy(data[off:off + rows * cols].reshape(rows, cols))
    assert np.array_equal(_bits(once[off:off + rows * cols]), _bits(want.ravel()))


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_is_refused_untouched(l2b, bad):
    w = (np.random.default_rng(3).standard_normal((4, 200)) * 0.1).astype(np.float32)
    w[3, 199] = bad
    before = w.copy()
    with pytest.raises(l2b.L2BError) as e:
        l2b.round_q8_host(w)
    assert e.value.status == -1
    assert np.array_equal(_bits(w), _bits(before))


def test_round_argument_checks(l2b):
    from llama2_zig_b200.binding import FP
    lib = l2b.load_library()
    n = C.c_uint64(7)
    w = np.ones((2, 4), np.float32)
    assert lib.l2b_round_q8_host(None, 2, 4, C.byref(n)) == -1
    assert lib.l2b_round_q8_host(w.ctypes.data_as(FP), 2, 0, C.byref(n)) == -1
    assert n.value == 7
    assert lib.l2b_round_q8_host(w.ctypes.data_as(FP), 2, 4, None) == 0      # the count is optional
    assert lib.l2b_round_q8_host(w.ctypes.data_as(FP), 0, 4, C.byref(n)) == 0 and n.value == 0
    with pytest.raises(TypeError):
        l2b.round_q8_host(np.zeros(8, np.float32))
    with pytest.raises(TypeError):
        l2b.round_q8_host(np.zeros((2, 4), np.float64))


def _has_device():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_format_checks_come_before_the_device(l2b):
    from llama2_zig_b200.binding import L2BConfig, FP
    lib = l2b.load_library()
    h = C.c_void_p()
    cfg = L2BConfig(288, 768, 6, 6, 6, 32000, 256, 1)
    n = int(lib.l2b_checkpoint_floats(C.byref(cfg)))
    data = np.zeros(n, np.float32)
    dp = data.ctypes.data_as(FP)
    for fmt in (2, 4, -1, 7):                              # unknown format (2 stays unknown)
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -1
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -1
        assert b"format" in lib.l2b_last_error(None)
    for fmt in (1, 3):                                     # bf16 and q8 are single-GPU
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 2, fmt) == -2
        assert b"single-GPU" in lib.l2b_last_error(None)
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), None, n, None, None, 1, fmt) == -1  # l2b_create's checks
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, 8, None, None, 1, fmt) == -1
        bad = L2BConfig(36, 768, 6, 6, 6, 32000, 256, 1)
        assert lib.l2b_create_format(C.byref(h), C.byref(bad), dp, n, None, None, 1, fmt) == -2
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(bad), 1, fmt) == -2
    assert not h.value
    if _has_device():
        return
    for fmt in (0, 1, 3):                                  # a valid call reaches the device check
        assert lib.l2b_create_format(C.byref(h), C.byref(cfg), dp, n, None, None, 1, fmt) == -4
        assert lib.l2b_create_synthetic_format(C.byref(h), C.byref(cfg), 1, fmt) == -4
    assert lib.l2b_weight_info(None, None, None) == -1


def test_oracle_quantization_cost_stories15m(oracle, l2b):
    """Greedy streams of the oracle on the stories15M-shaped fixture payload P and on dq(P): the first
    step where they part and the largest relative logit difference over the teacher-forced run."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    cfg = oracle.make_config(*oracle.STORIES15M_SHAPE)
    shared = True
    data = oracle.synth_checkpoint(cfg, shared, oracle.STORIES15M_SEED)
    ck = shape_checkpoint("stories15M")
    assert ck.shared_weights == shared
    dq, changed = dequant_matrices(l2b, ck, data)
    a = oracle.OracleModel(cfg, data, shared, W=8, kind="strict")
    b = oracle.OracleModel(cfg, dq, shared, W=8, kind="strict")
    steps = cfg.seq_len
    _, ga, _ = a.generate(1, steps, stop_on_bos=False)
    _, gb, _ = b.generate(1, steps, stop_on_bos=False)
    differ = np.nonzero(ga != gb)[0]
    first = int(differ[0]) if differ.size else None
    a.close(); b.close()
    a = oracle.OracleModel(cfg, data, shared, W=8, kind="strict")
    b = oracle.OracleModel(cfg, dq, shared, W=8, kind="strict")
    worst = 0.0
    tok = 1
    for pos in range(steps):
        la, lb = a.forward(tok, pos), b.forward(tok, pos)
        worst = max(worst, float(np.max(np.abs(la - lb)) / np.max(np.abs(la))))
        tok = int(ga[pos])
    a.close(); b.close()
    print(f"\nq8 quantization on stories15M-shaped seed {oracle.STORIES15M_SEED}: {changed} matrix weights "
          f"changed; greedy streams part at step {first} of {steps}; max relative logit difference {worst:.3e}")
    assert 0.0 < worst < 0.5
