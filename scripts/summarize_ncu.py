"""Turn Nsight Compute outputs into small markdown / JSON summaries (on any machine with ncu).

  python scripts/summarize_ncu.py launches launches_X.csv   > launches_X.md
  python scripts/summarize_ncu.py full     prof_X.ncu-rep   > ncu_X.md
  python scripts/summarize_ncu.py traffic  prof_X.ncu-rep WORKLOAD LABEL 'REGEX' SHA16 traffic.json
      (adds dram__bytes_read.sum + dram__bytes_write.sum per launch of the kernels matching REGEX as
       WORKLOAD/LABEL, tagged with the kernel-source sha the capture was built from)
"""
import collections
import csv
import subprocess
import sys


def launches(path):
    rows = list(csv.reader(open(path)))
    hi = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    h = rows[hi]
    ki, vi, gi = h.index("Kernel Name"), h.index("Metric Value"), h.index("Grid Size")
    agg = collections.OrderedDict()
    for r in rows[hi + 1:]:
        if len(r) <= vi:
            continue
        try:
            v = float(r[vi].replace(",", ""))
        except ValueError:
            continue
        a = agg.setdefault(r[ki], [0, 0.0, r[gi]])
        a[0] += 1
        a[1] += v
    tot = sum(a[1] for a in agg.values())
    print(f"# ncu launch list summary: `{path}`\n")
    print("`ncu --metrics gpu__time_duration.sum --clock-control none` — per-launch times are cold-cache and "
          "serialised; compare SHARES, not absolutes.\n")
    print("| kernel | launches | grid (last) | avg µs | share of GPU time |")
    print("|---|---|---|---|---|")
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"| `{k[:90]}` | {a[0]} | {a[2]} | {a[1] / a[0] / 1e3:.2f} | {a[1] / tot:.1%} |")
    print(f"\ntotal {tot / 1e3:.1f} µs over {sum(a[0] for a in agg.values())} launches")


WANT = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("dram__bytes_read.sum.per_second", "DRAM read rate"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM % of ncu peak"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 %"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("launch__registers_per_thread", "regs/thread"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem/block"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue active %"),
]


def full(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    h, units = rows[0], rows[1]
    print(f"# ncu --set full summary: `{path}`\n")
    print("| # | kernel | grid | " + " | ".join(n for _, n in WANT) + " | top stalls (warps per issue) |")
    print("|---|---|---|" + "---|" * (len(WANT) + 1))
    for i, r in enumerate(rows[2:]):
        cells = []
        for key, _ in WANT:
            if key in h:
                j = h.index(key)
                try:
                    cells.append(f"{float(r[j].replace(',', '')):.4g} {units[j]}")
                except ValueError:
                    cells.append(r[j])
            else:
                cells.append("-")
        stalls = []
        for name, val in zip(h, r):
            if name.startswith("smsp__average_warps_issue_stalled_") and name.endswith("_per_issue_active.ratio"):
                try:
                    stalls.append((float(val.replace(",", "")), name[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]))
                except ValueError:
                    pass
        stalls = ", ".join(f"{n} {v:.2f}" for v, n in sorted(stalls, reverse=True)[:4])
        print(f"| {i} | `{r[h.index('Kernel Name')][:60]}` | {r[h.index('Grid Size')]} | " + " | ".join(cells) + f" | {stalls} |")


def traffic(path, workload, label, regex, sha, out_json):
    import json
    import os
    import re
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    h = rows[0]
    ki, ri, wi = h.index("Kernel Name"), h.index("dram__bytes_read.sum"), h.index("dram__bytes_write.sum")
    units = rows[1]
    mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
    vals = []
    for r in rows[2:]:
        if re.search(regex, r[ki]):
            vals.append(float(r[ri].replace(",", "")) * mult[units[ri]] + float(r[wi].replace(",", "")) * mult[units[wi]])
    assert vals, f"no kernel matches {regex}"
    rec = json.load(open(out_json)) if os.path.exists(out_json) else {}
    if rec.get("kernel_source_sha16") != sha:
        rec = {"kernel_source_sha16": sha}
    rec.setdefault(workload, {})[label] = {"traffic": sum(vals) / len(vals), "launches": len(vals),
                                           "source": f"ncu --set full, {os.path.basename(path)}, kernels /{regex}/"}
    json.dump(rec, open(out_json, "w"), indent=1)
    print(workload, label, rec[workload][label])


if __name__ == "__main__":
    if sys.argv[1] == "traffic":
        traffic(*sys.argv[2:8])
    else:
        {"launches": launches, "full": full}[sys.argv[1]](sys.argv[2])
