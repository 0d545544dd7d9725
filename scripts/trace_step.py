"""In-kernel timeline of one llama2-7B decode step (graph + PDL), from %globaltimer stamps.
Run on the GPU box:  python scripts/trace_step.py [workload] [position] > trace.txt
Tensor parallel: launch it under torchrun (one process per GPU); rank 0 prints its own timeline.

The last part is the hand-off between consecutive kernels.  For each pair (A, B) it prints A's last
consumed slot (slot 5, max over CTAs; attention: its last epilogue, slot 7), B's entry (slot 0,
min..max) and B's first consumed slot (slot 4, min), and the window in which no SM consumes weights:
B's first consumption minus A's last (0 when they overlap).  The same window per SM (the ring GEMV
records its SM in slot 8) is averaged over the SMs both kernels ran on, and `early` counts the SMs
on which B's CTA entered before A's CTA there had consumed its last slot."""
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
last_pos = int(sys.argv[2]) if len(sys.argv) > 2 else 128
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
for pos in range(last_pos + 1):
    t.forward_argmax((1 + 7919 * pos) % ck.vocab_size, pos)
n_launch = 5 * L + 4
buf = np.zeros(n_launch * 512 * 16, dtype=np.uint64)
n = C.c_uint64()
rc = lib.l2b_debug_trace(t.h, buf.ctypes.data_as(C.POINTER(C.c_uint64)), buf.size, C.byref(n))
assert rc == 0, rc
slots = n.value // (n_launch * 512)
tr = buf[:n.value].reshape(n_launch, 512, slots).astype(np.int64)
# rows past a launch's grid, and slots a kernel does not stamp, may hold stamps of earlier launches
# (warm-up calls of the other step graphs): keep the stamps of the last step only
stamps = tr[:, :, :8]
stamps[stamps < stamps.max() - 100_000_000] = 0
tr[tr[:, :, 0] == 0] = 0
if rank != 0:
    t.close()
    dist.barrier()
    sys.exit(0)
names = ["qkv", "attn", "wo", "w13", "w2"]
stamps = tr[:, :, :8]
t0 = stamps[stamps > 0].min()
print(f"position {last_pos}")
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
step = (stamps[stamps > 0].max() - t0) / 1e3


# ---- hand-offs between consecutive kernels
def ctas(li):
    """CTAs of launch li that ran: their stamp rows (and SM ids when recorded)."""
    a = tr[li]
    live = a[:, 0] > 0
    return a[live]


def is_ring(a):
    return (a[:, 5] > 0).any()


def smid(a):
    return a[:, 8] if slots > 8 and is_ring(a) else None


def last_busy(a):
    """per CTA: its last consumed slot (ring GEMV) or its epilogue's end (attention)"""
    return a[:, 5] if is_ring(a) else a[:, 7]


hand = collections.defaultdict(list)
total_gap = 0.0
print("\nhand-offs [us since step start]: A last_cons(max) | B entry(min..max) first_cons(min) | gap  per-SM gap  early/SMs")
for li in range(5 * L):                                  # the last pair is (w2 of the last layer, classifier)
    A, B = ctas(li), ctas(li + 1)
    a_last = last_busy(A).max()
    b_first = B[:, 4][B[:, 4] > 0].min() if is_ring(B) else B[:, 2].min()
    gap = max(0.0, (b_first - a_last) / 1e3)
    total_gap += gap
    sa, sb = smid(A), smid(B)
    per_sm, early, common = float("nan"), 0, 0
    if sa is not None and sb is not None:
        la, fa = {}, {}
        for s, v in zip(sa, last_busy(A)):
            la[int(s)] = max(la.get(int(s), 0), int(v))
        eb, fb = {}, {}
        for s, e, f in zip(sb, B[:, 0], B[:, 4]):
            eb[int(s)] = min(eb.get(int(s), 1 << 62), int(e))
            fb[int(s)] = min(fb.get(int(s), 1 << 62), int(f))
        both = sorted(set(la) & set(eb))
        common = len(both)
        if both:
            per_sm = float(np.mean([max(0, fb[s] - la[s]) for s in both])) / 1e3
            early = sum(eb[s] < la[s] for s in both)
    kind = names[li % 5] + "->" + (names[(li + 1) % 5] if li + 1 < 5 * L else "cls")
    hand[kind].append((gap, per_sm, early, common))
    if li < 5 or li >= 5 * L - 5:
        print(f"{li:4d} {kind:10s} | {(a_last - t0) / 1e3:9.2f} | {(B[:, 0].min() - t0) / 1e3:8.2f}..{(B[:, 0].max() - t0) / 1e3:8.2f} "
              f"{(b_first - t0) / 1e3:9.2f} | {gap:6.2f} {per_sm:8.2f}  {early}/{common}")
print("\nper-kind hand-off averages over layers: gap [us]  per-SM gap [us]  SMs where B entered before A's last slot was consumed")
for k, v in hand.items():
    v = np.array(v, dtype=float)
    print(f"{k:10s} {np.mean(v[:, 0]):8.2f} {np.nanmean(v[:, 1]) if np.isfinite(v[:, 1]).any() else float('nan'):8.2f}"
          f"   {np.mean(v[:, 2]):6.1f} of {np.mean(v[:, 3]):5.1f}")
# SMs that ran two CTAs of one ring launch (the grid has one per SM; a doubled SM finishes late)
doubled = [int(np.max(np.bincount(smid(ctas(li))))) for li in range(5 * L + 1)
           if smid(ctas(li)) is not None and ctas(li).shape[0] > 0]
if doubled:
    print(f"most CTAs of one ring launch on one SM: {max(doubled)}  (launches with a doubled SM: {sum(d > 1 for d in doubled)} of {len(doubled)})")
print(f"\nstep span {step:.1f} us, hand-off gaps {total_gap:.1f} us ({100 * total_gap / step:.1f} % of the step)  (world {world})")
t.close()
if world > 1:
    dist.barrier()
