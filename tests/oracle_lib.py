"""ctypes view of the CPU parity oracle (oracle/build/liborc_{strict,fast}.so).

Test infrastructure only: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")


class OrcConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in
                ("dim", "hidden_dim", "n_layers", "n_heads", "n_kv_heads", "vocab_size", "seq_len")]


FP = C.POINTER(C.c_float)
IP = C.POINTER(C.c_int32)


def _fp(a):
    assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(FP)


def build_oracle():
    subprocess.run(["make", "-s", "-C", ORACLE_DIR], check=True)


_libs = {}


def load(kind="strict"):
    if kind in _libs:
        return _libs[kind]
    path = os.path.join(ORACLE_DIR, "build", f"liborc_{kind}.so")
    if not os.path.exists(path):
        build_oracle()
    lib = C.CDLL(path)
    lib.orc_matmul.argtypes = [FP, FP, FP, C.c_int, C.c_int, C.c_int]
    lib.orc_matmul_fused2.argtypes = [FP, FP, FP, FP, FP, C.c_int, C.c_int, C.c_int]
    lib.orc_matmul_fused3.argtypes = [FP, FP, FP, FP, FP, FP, FP, C.c_int, C.c_int, C.c_int]
    lib.orc_rmsnorm.argtypes = [FP, FP, FP, C.c_int, C.c_int]
    lib.orc_dot.argtypes = [FP, FP, C.c_int, C.c_int]
    lib.orc_dot.restype = C.c_float
    lib.orc_vector_mul.argtypes = [FP, FP, C.c_int, C.c_int]
    lib.orc_weighted_sum_rows.argtypes = [FP, C.c_int, FP, C.c_int, FP, C.c_int, C.c_int]
    lib.orc_softmax.argtypes = [FP, C.c_int]
    lib.orc_accum.argtypes = [FP, FP, C.c_int]
    lib.orc_argmax.argtypes = [FP, C.c_int]
    lib.orc_argmax.restype = C.c_int
    lib.orc_rope_angle.argtypes = [C.c_int, C.c_int, C.c_int, FP, FP]
    lib.orc_model_create.argtypes = [C.POINTER(OrcConfig), FP, C.c_int, C.c_int]
    lib.orc_model_create.restype = C.c_void_p
    lib.orc_model_destroy.argtypes = [C.c_void_p]
    lib.orc_transformer.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.orc_logits.argtypes = [C.c_void_p]
    lib.orc_logits.restype = FP
    lib.orc_state.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]
    lib.orc_state.restype = FP
    lib.orc_checkpoint_floats.argtypes = [C.POINTER(OrcConfig), C.c_int]
    lib.orc_checkpoint_floats.restype = C.c_uint64
    lib.orc_generate.argtypes = [C.c_void_p, C.c_int, C.c_int, IP, C.c_int, IP,
                                 C.POINTER(C.c_double)]
    lib.orc_generate.restype = C.c_int
    lib.orc_read_header.argtypes = [C.c_char_p, C.POINTER(OrcConfig), C.POINTER(C.c_int),
                                    C.POINTER(C.c_uint64)]
    lib.orc_read_payload.argtypes = [C.c_char_p, FP, C.c_uint64]
    lib.orc_synth_fill.argtypes = [FP, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double,
                                   C.c_double, C.c_float, C.c_float]
    lib.orc_synth_checkpoint.argtypes = [C.POINTER(OrcConfig), C.c_int, C.c_uint64, FP]
    _libs[kind] = lib
    return lib


STATE = {"x": 0, "xb": 1, "xb2": 2, "hb": 3, "hb2": 4, "q": 5, "k": 6, "v": 7, "att": 8,
         "key_cache": 9, "value_cache": 10}


def make_config(dim, hidden_dim, n_layers, n_heads, n_kv_heads, vocab_size, seq_len):
    return OrcConfig(dim, hidden_dim, n_layers, n_heads, n_kv_heads, vocab_size, seq_len)


class OracleModel:
    """Weights + RunState of the oracle (src/main.zig:53-162) over a float32 payload."""

    def __init__(self, cfg, data, shared_weights, W=8, kind="strict"):
        self.lib = load(kind)
        self.cfg = cfg
        self.data = np.ascontiguousarray(data, dtype=np.float32)  # keep alive (borrowed)
        need = self.lib.orc_checkpoint_floats(C.byref(cfg), int(shared_weights))
        assert self.data.size >= need, (self.data.size, need)
        self.h = self.lib.orc_model_create(C.byref(cfg), _fp(self.data), int(shared_weights), W)
        assert self.h, "orc_model_create failed"

    def close(self):
        if self.h:
            self.lib.orc_model_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def forward(self, token, pos):
        self.lib.orc_transformer(self.h, int(token), int(pos))
        return np.ctypeslib.as_array(self.lib.orc_logits(self.h), shape=(self.cfg.vocab_size,)).copy()

    def state(self, name):
        n = C.c_uint64()
        p = self.lib.orc_state(self.h, STATE[name], C.byref(n))
        return np.ctypeslib.as_array(p, shape=(n.value,)).copy()

    def generate(self, token0, n_steps, forced=None, stop_on_bos=True):
        out = np.full(n_steps, -1, dtype=np.int32)
        secs = C.c_double()
        fp = None
        if forced is not None:
            forced = np.ascontiguousarray(forced, dtype=np.int32)
            fp = forced.ctypes.data_as(IP)
        calls = self.lib.orc_generate(self.h, token0, n_steps, fp, int(stop_on_bos),
                                      out.ctypes.data_as(IP), C.byref(secs))
        return calls, out, secs.value


def read_checkpoint(path, kind="strict"):
    lib = load(kind)
    cfg = OrcConfig()
    shared = C.c_int()
    n = C.c_uint64()
    rc = lib.orc_read_header(path.encode(), C.byref(cfg), C.byref(shared), C.byref(n))
    if rc != 0:
        raise OSError(f"orc_read_header({path}) -> {rc}")
    data = np.empty(n.value, dtype=np.float32)
    rc = lib.orc_read_payload(path.encode(), _fp(data), n.value)
    if rc != 0:
        raise OSError(f"orc_read_payload({path}) -> {rc}")
    return cfg, bool(shared.value), data


def synth_checkpoint(cfg, shared_weights, seed, kind="strict"):
    lib = load(kind)
    n = lib.orc_checkpoint_floats(C.byref(cfg), int(shared_weights))
    data = np.empty(n, dtype=np.float32)
    lib.orc_synth_checkpoint(C.byref(cfg), int(shared_weights), seed, _fp(data))
    return data


# stories15M shape, synthetic weights.  Seed 10 keeps every greedy step's top-2 logit margin >= 0.016
# over all 256 positions (the shipped stories15M.bin has 0.0100), so free-running streams are stable.
STORIES15M_SHAPE = (288, 768, 6, 6, 6, 32000, 256)
STORIES15M_SEED = 10


def write_stories15m_checkpoint(path):
    """A stories15M-shaped llama2.c checkpoint file (28-byte header + payload, freq_cis included)."""
    cfg = make_config(*STORIES15M_SHAPE)
    data = synth_checkpoint(cfg, True, STORIES15M_SEED)
    with open(path, "wb") as f:
        f.write(np.array(STORIES15M_SHAPE, dtype="<i4").tobytes())
        f.write(data.astype("<f4").tobytes())
    return path


# stories15M shape with an unshared classifier (header vocab -32000), seed 10, classifier row 1 (BOS)
# scaled by 4: the greedy stream from BOS ends on BOS at position 19 (top-2 margin >= 0.098 at every
# step), so it exercises the BOS stop of src/main.zig:1017-1019.
BOS_STOP_SHAPE = (288, 768, 6, 6, 6, -32000, 256)
BOS_STOP_POS = 19


def bos_stop_payload():
    dim, vocab = BOS_STOP_SHAPE[0], -BOS_STOP_SHAPE[5]
    data = synth_checkpoint(make_config(*BOS_STOP_SHAPE[:5], vocab, BOS_STOP_SHAPE[6]), False, STORIES15M_SEED)
    wcls = data.size - vocab * dim
    data[wcls + dim:wcls + 2 * dim] *= 4.0
    return data
