"""CPU: pins the oracle against everything the reference's own tests hold for the hot path
(src/main.zig:1078-1150 of the reference) and against the committed golden fixtures."""
import hashlib
import json
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WIDTHS = (4, 8, 16)
KINDS = ("strict", "fast")


def fp(a):
    import ctypes as C
    return a.ctypes.data_as(C.POINTER(C.c_float))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("W", WIDTHS)
def test_matrix_multiplies(oracle, kind, W):
    """test "matrix_multiplies", src/main.zig:1078-1087 (exact equality)."""
    lib = oracle.load(kind)
    w = np.arange(1, 10, dtype=np.float32)
    x = np.array([1, 2, 3], dtype=np.float32)
    out = np.zeros(3, dtype=np.float32)
    lib.orc_matmul(fp(out), fp(x), fp(w), 3, 3, W)
    assert out[0] == 1.0 + 4.0 + 9.0
    assert out[1] == 4.0 + 10.0 + 18.0
    assert out[2] == 7.0 + 16.0 + 27.0


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("W", WIDTHS)
def test_vector_length_less_than_width_case(oracle, kind, W):
    """test "vector_length_less_than_width_case", src/main.zig:1089-1103 (exact vs scalar loop)."""
    lib = oracle.load(kind)
    w = np.arange(1, 25, dtype=np.float32)
    x = np.arange(1, 13, dtype=np.float32)
    out = np.zeros(2, dtype=np.float32)
    lib.orc_matmul(fp(out), fp(x), fp(w), 2, 12, W)
    for i in range(2):
        expected = np.float32(0)
        for j in range(12):
            expected = np.float32(expected + w[i * 12 + j] * x[j])
        assert out[i] == expected


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("W", WIDTHS)
def test_vector_weighted_sum_rows(oracle, kind, W):
    """test "vector_weighted_sum_rows", src/main.zig:1117-1139 (width W+3, stride W+5, abs 1e-5)."""
    lib = oracle.load(kind)
    width, stride = W + 3, W + 5
    weights = np.array([0.25, -0.5, 1.5], dtype=np.float32)
    rows = np.zeros(stride * 3, dtype=np.float32)
    for r in range(3):
        for i in range(width):
            rows[r * stride + i] = r * width + i + 1
    out = np.zeros(width, dtype=np.float32)
    lib.orc_weighted_sum_rows(fp(out), width, fp(rows), stride, fp(weights), 3, W)
    for i in range(width):
        expected = sum(float(rows[r * stride + i]) * float(weights[r]) for r in range(3))
        assert abs(expected - out[i]) <= 1e-5


@pytest.mark.parametrize("kind", KINDS)
def test_softmax(oracle, kind):
    """test "softmax", src/main.zig:1141-1150: {1,2,3,4} sums to exactly 1.0."""
    lib = oracle.load(kind)
    x = np.array([1, 2, 3, 4], dtype=np.float32)
    lib.orc_softmax(fp(x), 4)
    s = np.float32(0)
    for v in x:
        s = np.float32(s + v)
    assert s == 1.0


@pytest.mark.parametrize("W", WIDTHS)
def test_fused_matches_single_up_to_order(oracle, W):
    """matmul_fused(N=2|3) uses 4 accumulators, matmul 8 (src/main.zig:546): same value up to
    summation order, and each fused output equals a 4-accumulator evaluation of its own row."""
    lib = oracle.load("strict")
    rng = np.random.default_rng(0)
    d, n = 37, 8 * W + 5
    x = rng.standard_normal(n).astype(np.float32)
    ws = [rng.standard_normal(d * n).astype(np.float32) for _ in range(3)]
    single = [np.zeros(d, np.float32) for _ in range(3)]
    for o, w in zip(single, ws):
        lib.orc_matmul(fp(o), fp(x), fp(w), d, n, W)
    f3 = [np.zeros(d, np.float32) for _ in range(3)]
    lib.orc_matmul_fused3(fp(f3[0]), fp(f3[1]), fp(f3[2]), fp(x), fp(ws[0]), fp(ws[1]), fp(ws[2]), d, n, W)
    f2 = [np.zeros(d, np.float32) for _ in range(2)]
    lib.orc_matmul_fused2(fp(f2[0]), fp(f2[1]), fp(x), fp(ws[0]), fp(ws[1]), d, n, W)
    for j in range(3):
        np.testing.assert_allclose(f3[j], single[j], rtol=2e-5, atol=2e-5)
    for j in range(2):
        assert np.array_equal(f2[j], f3[j])  # same accumulator count => bit-identical


def test_rmsnorm_against_float64(oracle):
    lib = oracle.load("strict")
    rng = np.random.default_rng(1)
    for n in (3, 8, 288, 2988):  # 2988 = benchmarks/rmsnorm.zig size
        x = rng.standard_normal(n).astype(np.float32)
        w = rng.standard_normal(n).astype(np.float32)
        o = np.zeros(n, np.float32)
        lib.orc_rmsnorm(fp(o), fp(x), fp(w), n, 8)
        ref = x.astype(np.float64) / np.sqrt(np.mean(x.astype(np.float64) ** 2) + 1e-5) * w
        np.testing.assert_allclose(o, ref, rtol=3e-6, atol=1e-6)
        # in-place form used for the final norm (src/main.zig:426)
        xi = x.copy()
        lib.orc_rmsnorm(fp(xi), fp(xi), fp(w), n, 8)
        assert np.array_equal(xi, o)


def test_argmax_first_maximum_wins(oracle):
    lib = oracle.load("strict")
    x = np.array([0, 5, 5, 1], dtype=np.float32)
    assert lib.orc_argmax(fp(x), 4) == 1  # strict '>' (src/main.zig:720)


def test_golden_token_stream(oracle, stories15m):
    """configs[0]: the stories15M-shaped checkpoint, -t 0, 256 tokens on CPU."""
    with open(os.path.join(GOLDEN, "stories15M_t0_tokens.json")) as f:
        gold = json.load(f)
    assert gold["sha256_le_u32"] == "76f4096890fb99d6e0c8abca87b777dc9a20c8e47085da5d3ff50ed6dac7f808"
    cfg, shared, data = oracle.read_checkpoint(stories15m)
    assert (cfg.dim, cfg.hidden_dim, cfg.n_layers, cfg.n_heads, cfg.n_kv_heads, cfg.vocab_size,
            cfg.seq_len, shared) == (288, 768, 6, 6, 6, 32000, 256, True)
    assert os.path.getsize(stories15m) == gold["checkpoint_bytes"]
    m = oracle.OracleModel(cfg, data, shared, W=8, kind="strict")
    calls, out, _ = m.generate(1, 256)
    assert calls == gold["forward_calls"] == 256
    assert gold["terminator"] is None and 1 not in out[:calls]   # no BOS: the loop runs to seq_len (src/main.zig:1017-1019)
    toks = out[:calls]
    assert toks.tolist() == gold["tokens"]
    assert hashlib.sha256(toks.astype("<u4").tobytes()).hexdigest() == gold["sha256_le_u32"]


def test_generate_stops_on_bos(oracle):
    """BOS ends the loop (src/main.zig:1017-1019) on the position it is produced; without the stop the
    loop runs on to n_steps over the same prefix."""
    shape = oracle.BOS_STOP_SHAPE
    cfg = oracle.make_config(*shape[:5], -shape[5], shape[6])
    m = oracle.OracleModel(cfg, oracle.bos_stop_payload(), False, W=8, kind="strict")
    calls, out, _ = m.generate(1, 256)
    k = oracle.BOS_STOP_POS
    assert calls == k + 1 and out[k] == 1 and 1 not in out[:k].tolist()
    m2 = oracle.OracleModel(cfg, oracle.bos_stop_payload(), False, W=8, kind="strict")
    calls2, out2, _ = m2.generate(1, 256, stop_on_bos=False)
    assert calls2 == 256 and np.array_equal(out2[:k + 1], out[:k + 1])


def test_golden_logits_fixture(oracle, stories15m):
    gold = np.load(os.path.join(GOLDEN, "stories15M_logits.npz"))
    with open(os.path.join(GOLDEN, "stories15M_t0_tokens.json")) as f:
        toks = json.load(f)["tokens"] + [1]
    cfg, shared, data = oracle.read_checkpoint(stories15m)
    m = oracle.OracleModel(cfg, data, shared, W=8, kind="strict")
    token = 1
    for pos in range(int(gold["positions"].max()) + 1):
        lg = m.forward(token, pos)
        if pos in gold["positions"]:
            assert np.array_equal(lg[::16], gold[f"p{pos}_strided"])
            assert np.array_equal(lg[gold[f"p{pos}_top_idx"]], gold[f"p{pos}_top_val"])
        token = toks[pos]


def test_synth_generator_matches_product_host_mirror(oracle, l2b):
    """The oracle's synthetic-checkpoint generator and the product's host mirror (which is
    bit-identical to the device generator, checked in the gpu tests) must agree exactly."""
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint((64, 172, 2, 4, 2, 96, 32))           # shared classifier, GQA
    a = oracle.synth_checkpoint(oracle.make_config(*ck.shape_tuple), True, 7)
    b = l2b.synth_checkpoint_host(ck, 7)
    assert a.size == b.size == l2b.checkpoint_floats(ck)
    assert np.array_equal(a, b)
    ck2 = shape_checkpoint((64, 172, 2, 4, 4, -96, 32))         # unshared classifier
    a2 = oracle.synth_checkpoint(oracle.make_config(*ck2.shape_tuple), False, 9)
    b2 = l2b.synth_checkpoint_host(ck2, 9)
    assert np.array_equal(a2, b2) and a2.size == a.size - 0 + 96 * 64 + (2 * 64 * 64 - 2 * 64 * 32) * 2
    # distribution sanity: rms gains are clipped to [0.25, 2.4], embeddings ~ N(0, 0.04)
    emb = a[:96 * 64]
    assert abs(float(emb.std()) - 0.04) < 0.004
    gains = a[96 * 64:96 * 64 + 2 * 64]
    assert gains.min() >= 0.25 and gains.max() <= 2.4
