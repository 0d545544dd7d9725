"""In-kernel timeline of one llama2-7B decode step (graph + PDL), from %globaltimer stamps.
Run on the GPU box:  python scripts/trace_step.py [workload] > trace.txt
Tensor parallel: launch it under torchrun (one process per GPU); rank 0 prints its own timeline."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["L2B_TRACE"] = "1"
import llama2_zig_b200 as l2b
from llama2_zig_b200.checkpoint import shape_checkpoint

wl = sys.argv[1] if len(sys.argv) > 1 else "llama2-7B"
ck = shape_checkpoint(wl)
rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
if world > 1:
    import torch
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    idt = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        idt.copy_(torch.frombuffer(bytearray(l2b.comm_unique_id()), dtype=torch.uint8))
    dist.broadcast(idt, 0)
    t = l2b.Transformer(ck, synthetic_seed=7, rank=rank, world_size=world, device=local,
                        comm_id=bytes(idt.cpu().numpy().tobytes()))
else:
    t = l2b.Transformer(ck, synthetic_seed=7)
lib = l2b.load_library()
lib.l2b_debug_trace.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint64)]
L = ck.n_layers
for pos in range(40):
    t.forward_argmax((1 + 7919 * pos) % ck.vocab_size, pos)
n_launch = 5 * L + 4
buf = np.zeros(n_launch * 512 * 8, dtype=np.uint64)
n = C.c_uint64()
rc = lib.l2b_debug_trace(t.h, buf.ctypes.data_as(C.POINTER(C.c_uint64)), buf.size, C.byref(n))
assert rc == 0, rc
tr = buf.reshape(n_launch, 512, 8).astype(np.int64)
if rank != 0:
    t.close()
    dist.barrier()
    sys.exit(0)
names = ["qkv", "attn", "wo", "w13", "w2"]
t0 = tr[tr > 0].min()
print("launch kernel  | entry(min..max) ring_filled  wait_done(min..max)  staged(max)  first_cons(min)  last_cons(max)  prod_done(max)  epi_done(max)   [us since step start]")
prev_end = 0
for li in range(5 * L + 1):
    name = names[li % 5] + f"{li // 5}" if li < 5 * L else "cls"
    a = tr[li]
    def mm(slot, f):
        v = a[:, slot]
        v = v[v > 0]
        return (f(v) - t0) / 1e3 if v.size else float("nan")
    if li < 10 or li >= 5 * L - 5 or (25 <= li < 30):
        print(f"{li:4d} {name:7s} | {mm(0,np.min):8.2f}..{mm(0,np.max):8.2f} {mm(1,np.max):9.2f}   {mm(2,np.min):8.2f}..{mm(2,np.max):8.2f} {mm(3,np.max):9.2f} {mm(4,np.min):12.2f} {mm(5,np.max):14.2f} {mm(6,np.max):14.2f} {mm(7,np.max):14.2f}")
# per-kind averages of the interesting gaps over all layers
import collections
agg = collections.defaultdict(list)
for li in range(5 * L):
    a = tr[li]
    def mx(slot):
        v = a[:, slot]; v = v[v > 0]; return v.max() if v.size else 0
    def mn(slot):
        v = a[:, slot]; v = v[v > 0]; return v.min() if v.size else 0
    kind = names[li % 5]
    if kind == "attn":
        agg[kind].append(((mx(7) - mn(0)) / 1e3, (mn(2) - mn(0)) / 1e3, 0, 0, 0))
    else:
        # duration entry->epi_done, wait (entry->wait_done max), staging (wait_done->staged), stream (first_cons->last_cons), tail (last_cons->epi_done)
        agg[kind].append(((mx(7) - mn(0)) / 1e3, (mx(2) - mn(0)) / 1e3, (mx(3) - mx(2)) / 1e3, (mx(5) - mn(4)) / 1e3, (mx(7) - mx(5)) / 1e3))
print("\nper-kind averages over layers [us]: total(entry_min->epi_max)  entry->wait_done  wait_done->staged  first->last consume  last consume->epilogue done")
for k, v in agg.items():
    v = np.array(v)
    print(f"{k:5s}", " ".join(f"{x:8.2f}" for x in v.mean(axis=0)))
step = (tr[tr > 0].max() - t0) / 1e3
print(f"\nstep span {step:.1f} us  (world {world})")
t.close()
if world > 1:
    dist.barrier()
