"""Phase timeline of the all-layers cluster kernel (stories15M-class models): L2B_TRACE stamps of CTA 0."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["L2B_TRACE"] = "1"
import llama2_zig_b200 as l2b
from llama2_zig_b200.checkpoint import shape_checkpoint

ck = shape_checkpoint(sys.argv[1] if len(sys.argv) > 1 else "stories15M")
t = l2b.Transformer(ck, synthetic_seed=7)
lib = l2b.load_library()
lib.l2b_debug_trace.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint64)]
for pos in range(40):
    t.forward_argmax((1 + 7919 * pos) % ck.vocab_size, pos)
n_launch = 5 * ck.n_layers + 4
buf = np.zeros(n_launch * 512 * 16, dtype=np.uint64)
n = C.c_uint64()
assert lib.l2b_debug_trace(t.h, buf.ctypes.data_as(C.POINTER(C.c_uint64)), buf.size, C.byref(n)) == 0
st = buf[:ck.n_layers * 32].reshape(ck.n_layers, 32).astype(np.int64)
names = ["start", "p1 qkv done", "sync1", "p2 attn done", "sync2", "p3 wo done", "sync3", "gather x", "p4 w13 done", "sync4",
         "p5 w2 done", "sync5", "gather x"]
print("phase deltas [us] per layer (CTA 0 of the cluster)")
print("layer " + " ".join(f"{n_:>12s}" for n_ in names[1:]) + "        total")
for l in range(ck.n_layers):
    d = [(st[l, k] - st[l, k - 1]) / 1e3 for k in range(1, 13)]
    print(f"{l:5d} " + " ".join(f"{v:12.2f}" for v in d) + f" {(st[l, 12] - st[l, 0]) / 1e3:12.2f}")
print("\nsub-phases [us]: p1: rmsnorm | dot+rope+store | issue next | fence ;  p2: q gather | kv loop | merge | out ;  p4: rmsnorm | tiles | issue")
for l in range(ck.n_layers):
    a = st[l]
    print(f"{l:5d} p1 {(a[16]-a[0])/1e3:6.2f} {(a[17]-a[16])/1e3:6.2f} {(a[18]-a[17])/1e3:6.2f} {(a[1]-a[18])/1e3:6.2f} ; "
          f"p2 {(a[19]-a[2])/1e3:6.2f} {(a[20]-a[19])/1e3:6.2f} {(a[21]-a[20])/1e3:6.2f} {(a[3]-a[21])/1e3:6.2f} ; "
          f"p4 {(a[22]-a[7])/1e3:6.2f} {(a[23]-a[22])/1e3:6.2f} {(a[8]-a[23])/1e3:6.2f}")
t.close()
