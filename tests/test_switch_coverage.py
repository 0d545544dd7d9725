"""CPU: every run-time switch the CUDA library reads is documented and exercised on the GPU.

Collects each getenv("L2B_...") under llama2.zig_b200/csrc/ and requires it both in the run-time
switch table of DESIGN.md §7 and in tests/test_gpu_variants.py, so a new switch cannot ship with
its kernel path untested or undocumented."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# switches that select no kernel and change no arithmetic
EXEMPT = {
    "L2B_TRACE": "adds %globaltimer stamps to every kernel; the results are those of the untraced kernels",
    "L2B_SPIN_TIMEOUT_MS": "bounds the tensor-parallel peer waits only",
    "L2B_TP": "tensor parallel only (tests/test_gpu_tp.py needs several GPUs)",
}


def library_switches():
    names = set()
    for path in glob.glob(os.path.join(ROOT, "llama2.zig_b200", "csrc", "*.cu*")):
        with open(path) as f:
            names |= set(re.findall(r'getenv\(\s*"(L2B_[A-Z0-9_]+)"\s*\)', f.read()))
    return names


def design_switch_table():
    with open(os.path.join(ROOT, "DESIGN.md")) as f:
        text = f.read()
    section = re.search(r"^## 7\..*?(?=^## )", text, flags=re.S | re.M)
    assert section, "DESIGN.md has no §7"
    rows = [line for line in section.group(0).splitlines() if line.startswith("|")]
    return set(re.findall(r"`(L2B_[A-Z0-9_]+)", "\n".join(rows)))


def test_library_reads_switches():
    names = library_switches()
    assert {"L2B_NO_GRAPH", "L2B_FUSE", "L2B_ATTN"} <= names, names   # the scan itself works


def test_every_switch_is_documented():
    missing = sorted(library_switches() - design_switch_table())
    assert not missing, f"not in the DESIGN.md §7 table: {missing}"


def test_every_switch_is_exercised_by_the_variant_module():
    with open(os.path.join(ROOT, "tests", "test_gpu_variants.py")) as f:
        text = f.read()
    used = set(re.findall(r"\b(L2B_[A-Z0-9_]+)\b", text))
    missing = sorted(library_switches() - set(EXEMPT) - used)
    assert not missing, f"no case in tests/test_gpu_variants.py sets: {missing}"
    assert set(EXEMPT) <= library_switches(), "stale exemption"
