#!/usr/bin/env python
"""Prints a markdown excerpt: per hot kernel of libllama2_b200.so, the SASS mnemonics that
prove the Hopper-native mechanisms (VERDICT r1 #9): UBLKCP = cp.async.bulk (TMA bulk copy),
SYNCS = mbarrier ops, ACQBULK/PREEXIT = griddepcontrol.wait / launch_dependents (PDL),
LDG.E.128 / LDS.128 = 128-bit loads, STG/LDG.E.128.STRONG.SYS = the LL units that cross NVLink.
Needs no GPU: `python scripts/sass_excerpt.py TAG > sass_excerpt.md`."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "llama2.zig_b200", "lib", "libllama2_b200.so")
tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
elf = subprocess.run(["cuobjdump", "-lelf", LIB], capture_output=True, text=True).stdout
funcs, cur = collections.OrderedDict(), None
for line in sass.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        cur = m.group(1)
        funcs[cur] = []
    elif cur and "/*" in line and ";" in line:
        funcs[cur].append(line)
names = subprocess.run(["c++filt"] + list(funcs), capture_output=True, text=True).stdout.splitlines()
PATS = [("UBLKCP", r"\bUBLKCP"), ("SYNCS (mbarrier)", r"\bSYNCS"), ("ACQBULK (griddepcontrol.wait)", r"\bACQBULK"),
        ("PREEXIT (launch_dependents)", r"\bPREEXIT"), ("LDG.E.128", r"\bLDG\.E\.128"), ("LDS.128", r"\bLDS\.128"),
        ("FFMA", r"\bFFMA"), ("SHFL", r"\bSHFL"), ("ST.*.SYS (LL store)", r"\bSTG\.E\.128\.STRONG\.SYS"),
        ("LD.*.SYS (LL load)", r"\bLDG\.E\.128\.STRONG\.SYS"), ("HMMA/UTC*MMA (must be 0)", r"\b(HMMA|UTC\w*MMA|HGMMA)")]
HOT = ["gemv_tma_kernel<2>", "gemv_tma_kernel<3>", "gemv_tma_kernel<5>", "gemv_tma_kernel<4>", "gemv_tma_kernel<0>",
       "gemv_tma_kernel<1>", "gemv_kernel<32, 2>", "gemv_kernel<8, 1>", "attention_flash_kernel<3>",
       "attention_flash_kernel<8>", "attn_wo_kernel", "ffn_fused_kernel", "advance_kernel", "gather_logits_kernel",
       "sample_prep_kernel"]
out = [f"# SASS evidence, {tag} (cuobjdump -sass llama2.zig_b200/lib/libllama2_b200.so; single sm_90a cubin)", "",
       "ELF list: " + ", ".join(l.split()[-1] for l in elf.splitlines() if "sm_" in l), "",
       "Counts of the mnemonics that matter per hot kernel (EPI template index: 0 store, 1 argmax, 2 qkv+rope, "
       "3 silu, 4 tensor-parallel LL exchange, 5 residual add):", "",
       "| kernel | " + " | ".join(p[0] for p in PATS) + " | instructions |", "|---|" + "---|" * (len(PATS) + 1)]
picked = []
for raw, nm in zip(funcs, names):
    short = nm.replace("l2b::", "").replace("(l2b::GemvParams)", "").replace("void ", "")
    if any(h in short for h in HOT):
        body = funcs[raw]
        row = [str(sum(1 for l in body if re.search(p[1], l))) for p in PATS]
        out.append(f"| `{short[:60]}` | " + " | ".join(row) + f" | {len(body)} |")
        picked.append((short, body))
out += ["", "## Excerpts (first occurrence of each mechanism in `gemv_tma_kernel<3>`, the w13_silu kernel)", "", "```"]
for short, body in picked:
    if "gemv_tma_kernel<3>" in short:
        for label, pat in PATS[:6]:
            for l in body:
                if re.search(pat, l):
                    out.append(l.rstrip()[:150])
                    break
        break
out += ["```", "", "## LL exchange (`gemv_tma_kernel<4>` stores, `tp_reduce_into_x` loads inside `gemv_tma_kernel<3>`)", "", "```"]
for short, body in picked:
    if "gemv_tma_kernel<4>" in short:
        out += [l.rstrip()[:150] for l in body if re.search(r"\bSTG\.E\.128\.STRONG\.SYS", l)][:2]
    if "gemv_tma_kernel<3>" in short:
        out += [l.rstrip()[:150] for l in body if re.search(r"\bLDG\.E\.128\.STRONG\.SYS", l)][:2]
out += ["```", ""]
print("\n".join(out))
