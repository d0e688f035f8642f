#!/usr/bin/env python
"""Opcode histogram of the tensor-core kernels in libzsb200.so (cuobjdump -sass): evidence that the
hot kernels are wgmma / TMA code (HGMMA = wgmma.mma_async, WARPGROUP.ARRIVE = wgmma.fence,
WARPGROUP.DEPBAR = wgmma.wait_group, UTMALDG = TMA tensor load, SYNCS = mbarrier ops).  A healthy
mainloop has about one WARPGROUP.DEPBAR per k-block loop, not one per HGMMA.  Writes a markdown
table."""
import collections
import re
import subprocess
import sys

so = sys.argv[1] if len(sys.argv) > 1 else "zhusuan_b200/libzsb200.so"
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
KEEP = ("HGMMA", "WARPGROUP.DEPBAR", "WARPGROUP.ARRIVE", "UTMALDG", "UTMAPF", "SYNCS", "BAR",
        "LDG", "STG", "LDS", "STS", "SHFL", "FFMA", "FMUL", "FADD", "F2FP", "MUFU", "FENCE",
        "RED", "ATOM", "MEMBAR", "CCTL")
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


def short(name):
    return re.sub(r"\(.*", "", name.replace("(anonymous namespace)::", "").replace("void ", ""))


print("| kernel | instr | " + " | ".join(KEEP[:12]) + " |")
print("|---|---:|" + "---:|" * 12)
for f, name in zip(hist, demangle):
    c = hist[f]
    if not any(k.startswith(("HGMMA", "UTMALDG")) for k in c):
        continue
    fam = collections.Counter()
    for k, v in c.items():
        for p in KEEP:
            if k == p or k.startswith(p + "."):
                fam[p] += v
                break
    print("| `%s` | %d | %s |" % (short(name), sum(c.values()), " | ".join(str(fam[p]) for p in KEEP[:12])))
print()
print("Full-opcode detail of the flagship kernel (the 49 middle passes of a dense_impl 5 trajectory):")
for f, name in zip(hist, demangle):
    if "tc_pipeline_kernel<(anonymous namespace)::ResW<0, 1, 1024, 2, 2> >" in name:
        c = hist[f]
        print("\n`%s`" % short(name))
        print(", ".join("%s x%d" % kv for kv in sorted(c.items(), key=lambda kv: -kv[1])
                        if kv[0].startswith(("HGMMA", "WARPGROUP", "UTMA", "SYNCS", "FENCE", "RED",
                                             "MEMBAR", "CCTL", "BAR"))))
