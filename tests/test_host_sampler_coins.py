"""CPU: the host twin's samplers with an explicit coin (l2h_sample_r, l2h_sample_top_p_r,
l2h_sample_top_p_candidates_r).  The PRNG forms draw one coin and call the coin form, except that
l2h_sample_top_p draws nothing when no entry passes the cutoff (src/main.zig:761-768 leaves nothing to walk).
Sampled speculative decoding relies on both: the host walks the target's positions with the coin forms and
must consume coins exactly as the plain loop does.

  * the PRNG forms give the streams in tests/golden/host_sampler_streams.json, which were recorded from the
    sampler before the coin forms existed: same seed, same tokens, for top-p in {0, 0.5, 0.9, 1} on random
    probability vectors with an all-below-cutoff vector every seventh step;
  * the coin forms, fed the generator's coins in order and skipping the coin where nothing passes the
    cutoff, give the same streams.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP = C.POINTER(C.c_float)
N = 64
TOP_PS = (0.0, 0.5, 0.9, 1.0)
SEED = 1234
M64 = (1 << 64) - 1


class PI(C.Structure):
    _fields_ = [("prob", C.c_float), ("index", C.c_int32)]


def vectors(count=60):
    """Random probability vectors of N entries; every seventh is flat below every cutoff used here."""
    rng = np.random.default_rng(11)
    for i in range(count):
        if i % 7 == 3:
            yield np.full(N, np.float32(1e-4), dtype=np.float32)
        else:
            u = rng.random(N).astype(np.float32) ** 4
            yield (u / u.sum(dtype=np.float32)).astype(np.float32)


def coins(seed):
    """The twin's PRNG (xoshiro256++ seeded through splitmix64, 24-bit float mapping): its uniform draws."""
    s = []
    for _ in range(4):
        seed = (seed + 0x9E3779B97F4A7C15) & M64
        z = seed
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        s.append(z ^ (z >> 31))
    rotl = lambda x, k: ((x << k) | (x >> (64 - k))) & M64   # noqa: E731
    while True:
        r = (rotl((s[0] + s[3]) & M64, 23) + s[0]) & M64
        t = (s[1] << 17) & M64
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]   # noqa: E702
        s[2] ^= t
        s[3] = rotl(s[3], 45)
        yield float(np.float32(r >> 40) * np.float32(1.0 / 16777216.0))


@pytest.fixture(scope="module")
def host():
    path = os.path.join(ROOT, "llama2.zig_b200", "lib", "libllama2_host.so")
    if not os.path.exists(path):
        pytest.skip("host twin not built")
    C.CDLL(os.path.join(ROOT, "llama2.zig_b200", "lib", "libllama2_b200.so"), mode=C.RTLD_GLOBAL)
    lib = C.CDLL(path)
    lib.l2h_sample.argtypes = [FP, C.c_int32]
    lib.l2h_sample_top_p.argtypes = [FP, C.c_int32, C.c_float, C.c_void_p]
    lib.l2h_sample_top_p_candidates.argtypes = [C.POINTER(PI), C.c_int32, C.c_float]
    lib.l2h_sample_r.argtypes = [FP, C.c_int32, C.c_float]
    lib.l2h_sample_top_p_r.argtypes = [FP, C.c_int32, C.c_float, C.c_void_p, C.c_float]
    lib.l2h_sample_top_p_candidates_r.argtypes = [C.POINTER(PI), C.c_int32, C.c_float, C.c_float]
    lib.l2h_seed.argtypes = [C.c_uint64]
    return lib


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "host_sampler_streams.json")) as f:
        return json.load(f)


def candidates(v, p):
    cut = np.float32((np.float32(1) - np.float32(p)) / (np.float32(N) - np.float32(1)))
    keep = np.nonzero(v >= cut)[0]
    return (PI * max(keep.size, 1))(*[PI(float(v[i]), int(i)) for i in keep]), keep.size


@pytest.mark.parametrize("kind", ["full", "candidates"])
@pytest.mark.parametrize("p", TOP_PS)
def test_prng_forms_keep_their_streams(host, golden, p, kind):
    host.l2h_seed(SEED)
    got = []
    scratch = (C.c_uint64 * N)()
    for v in vectors():
        cand, m = candidates(v, p)
        if p in (0.0, 1.0):
            got.append(host.l2h_sample(v.ctypes.data_as(FP), N))
        elif kind == "full" or m == 0:
            got.append(host.l2h_sample_top_p(v.ctypes.data_as(FP), N, p, scratch))
        else:
            got.append(host.l2h_sample_top_p_candidates(cand, m, p))
    assert got == golden[f"{p}/{kind}"]


@pytest.mark.parametrize("kind", ["full", "candidates"])
@pytest.mark.parametrize("p", TOP_PS)
def test_coin_forms_give_the_same_streams(host, golden, p, kind):
    draw = coins(SEED)
    coin = next(draw)
    got, skipped = [], 0
    scratch = (C.c_uint64 * N)()
    for v in vectors():
        cand, m = candidates(v, p)
        if p in (0.0, 1.0):
            got.append(host.l2h_sample_r(v.ctypes.data_as(FP), N, coin))
        elif m == 0:                                   # nothing passes: the argmax, the coin stays
            got.append(host.l2h_sample_top_p_r(v.ctypes.data_as(FP), N, p, scratch, coin))
            assert got[-1] == int(np.argmax(v))
            skipped += 1
            continue
        elif kind == "full":
            got.append(host.l2h_sample_top_p_r(v.ctypes.data_as(FP), N, p, scratch, coin))
        else:
            got.append(host.l2h_sample_top_p_candidates_r(cand, m, p, coin))
        coin = next(draw)
    assert got == golden[f"{p}/{kind}"]
    assert skipped == (0 if p in (0.0, 1.0) else 9)
