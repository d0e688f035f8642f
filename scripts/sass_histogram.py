#!/usr/bin/env python
"""Opcode histogram of the tensor-core kernels in libzsb200.so (cuobjdump -sass): evidence that the
hot kernels are wgmma / TMEM / TMA code (UTCHMMA = wgmma.mma, UTMALDG = TMA tensor load, LDTM =
wgmma.ld, UTCBAR = wgmma.commit, SYNCS = mbarrier ops).  Writes a markdown table."""
import collections
import re
import subprocess
import sys

so = sys.argv[1] if len(sys.argv) > 1 else "zhusuan_b200/libzsb200.so"
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
KEEP = ("UTCHMMA", "UTCQMMA", "UTMALDG", "UTMASTG", "UTMAPF", "LDTM", "UTCBAR", "UTCATOMSWS",
        "SYNCS", "FENCE", "RED", "ATOM", "LDG", "STG", "LDS", "STS", "FFMA", "FMUL", "FADD", "F2FP",
        "F2F", "HADD2", "MUFU", "SHFL", "BAR", "CCTL", "ERRBAR", "MEMBAR", "NANOSLEEP", "UCGABAR")
fn = None
hist = collections.OrderedDict()
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        fn = m.group(1)
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?PT?\d*\s+)?([A-Z][A-Z0-9_.]+)", line)
    if m and fn:
        hist.setdefault(fn, collections.Counter())[m.group(1)] += 1
demangle = subprocess.run(["c++filt"], input="\n".join(hist), capture_output=True, text=True).stdout.split("\n")
print("| kernel | instr | " + " | ".join(KEEP[:12]) + " |")
print("|---|---:|" + "---:|" * 12)
for f, name in zip(hist, demangle):
    c = hist[f]
    if not any(k.startswith(("UTCHMMA", "UTMALDG", "LDTM")) for k in c):
        continue
    short = re.sub(r"\(.*", "", name.replace("(anonymous namespace)::", "").replace("void ", ""))
    fam = collections.Counter()
    for k, v in c.items():
        for p in KEEP:
            if k == p or k.startswith(p + "."):
                fam[p] += v
                break
    print("| `%s` | %d | %s |" % (short, sum(c.values()), " | ".join(str(fam[p]) for p in KEEP[:12])))
print()
print("Full-opcode detail of the flagship kernels:")
for f, name in zip(hist, demangle):
    if "dense_res_kernel<1024, 0>" in name or "dense_leapfrog_tc2_kernel<32, 0, 1, 1, 1024>" in name:
        c = hist[f]
        print("\n`%s`" % re.sub(r"\(.*", "", name.replace("(anonymous namespace)::", "").replace("void ", "")))
        print(", ".join("%s x%d" % kv for kv in sorted(c.items(), key=lambda kv: -kv[1])
                        if kv[0].startswith(("UT", "LDTM", "SYNCS", "FENCE", "RED", "UCGABAR", "MEMBAR", "CCTL", "NANOSLEEP"))))
