"""Per-kernel SASS instruction counts of libmatchering_b200.so (cuobjdump -sass): TMA bulk copies (UBLKCP), mbarrier
operations (SYNCS), block barriers (BAR), FP32 / FP64 arithmetic, shared-memory and global loads/stores, warp
shuffles, tensor-core instructions (none expected).  Runs without a GPU.   python tools/sass_counts.py > profiles/rNN_sass_counts.txt"""
import os
import re
import subprocess
import sys
from collections import Counter, OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "matchering_b200", "libmatchering_b200.so")
GROUPS = OrderedDict([
    ("UBLKCP", r"^UBLKCP"), ("SYNCS", r"^SYNCS"), ("BAR", r"^BAR"), ("FFMA", r"^FFMA"), ("FADD", r"^FADD"), ("FMUL", r"^FMUL"),
    ("FFMA2/FADD2/FMUL2", r"^F(FMA|ADD|MUL)2"), ("DFMA", r"^DFMA"), ("DADD", r"^DADD"), ("DMUL", r"^DMUL"), ("MUFU", r"^MUFU"),
    ("LDS", r"^LDS"), ("STS", r"^STS"), ("LDG", r"^LDG"), ("STG", r"^STG"), ("SHFL", r"^SHFL"), ("ATOM/RED", r"^(ATOM|RED)"),
    ("tensor (HMMA/UTC*MMA)", r"^(HMMA|IMMA|DMMA|UTC.*MMA|QGMMA|HGMMA)"),
])
sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
demangle = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()


def without_parameters(name):
    """Cut the parameter list: the first '(' outside the template brackets (template arguments such as
    `(MeanMode)1` keep their parentheses, so every instantiation keeps its own row)."""
    depth = 0
    for i, ch in enumerate(name):
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            return name[:i]
    return name



kernels, current = OrderedDict(), None
arch = re.search(r"arch = (sm_\w+)", sass)
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = demangle(m.group(1))
        name = name.replace("void ", "").replace("mgb::", "").replace("(anonymous namespace)::", "")
        name = without_parameters(name)
        current = kernels.setdefault(name, Counter())
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
    if m and current is not None:
        op = m.group(1)
        current["total"] += 1
        for label, pat in GROUPS.items():
            if re.match(pat, op):
                current[label] += 1
print(f"# {os.path.relpath(LIB, ROOT)}: arch = {arch.group(1) if arch else '?'}; static SASS instruction counts per kernel")
cols = ["total"] + list(GROUPS)
print("kernel".ljust(58) + " ".join(c.rjust(9) for c in cols))
want = sys.argv[1:] or None
for name, c in kernels.items():
    if name.startswith("test_fft_kernel") or (want and not any(w in name for w in want)):
        continue
    print(name[:57].ljust(58) + " ".join(str(c.get(k, 0)).rjust(9) for k in cols))
tot = Counter()
for c in kernels.values():
    tot.update(c)
print("ALL KERNELS (incl. test harness)".ljust(58) + " ".join(str(tot.get(k, 0)).rjust(9) for k in cols))
