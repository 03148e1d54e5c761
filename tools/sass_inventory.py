#!/usr/bin/env python
"""SASS / resource inventory of libmacaw_b200.so (no GPU needed: `cuobjdump` reads the cubin nvcc cross-compiled).

Per kernel: registers, static + dynamic-independent shared memory, local (spill) bytes, and how often the Hopper
mnemonics that prove a wgmma / TMA / mbarrier kernel appear (HGMMA = wgmma.mma_async: HGMMA on 16-bit, QGMMA on e4m3 operands, UTMALDG = TMA tensor load,
SYNCS = mbarrier operations, WARPGROUP = warpgroup arrive / wait) next to HMMA (mma.sync).
Usage: python tools/sass_inventory.py
"""
import os
import re
import subprocess
import sys
from collections import OrderedDict, defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "macaw-llm_b200", "libmacaw_b200.so")

COLS = OrderedDict([
    ("HGMMA", r"\b[HQ]GMMA\."), ("UTMALDG", r"\bUTMALDG"), ("SYNCS", r"\bSYNCS\."), ("WARPGROUP", r"\bWARPGROUP\."),
    ("HMMA", r"\bHMMA\."), ("MUFU.EX2", r"\bMUFU\.EX2"),
])


def run(*cmd):
    return subprocess.run(cmd, check=True, capture_output=True, text=True).stdout


def demangle(names):
    out = run("c++filt", *names).splitlines()
    short = []
    for n in out:
        n = re.sub(r"^void ", "", n).replace("(anonymous namespace)::", "")
        n = re.sub(r"\(.*$", "", n)  # drop the parameter list
        short.append(n.replace("mm::", ""))
    return dict(zip(names, short))


def main():
    if not os.path.exists(LIB):
        sys.exit(f"{LIB} missing: run `python __graft_entry__.py` first")
    sass = run("cuobjdump", "-sass", LIB)
    counts = defaultdict(lambda: defaultdict(int))
    fn = None
    pats = {k: re.compile(v) for k, v in COLS.items()}
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            counts[fn]  # touch
            continue
        if fn is None or "/*" not in line:
            continue
        for k, p in pats.items():
            if p.search(line):
                counts[fn][k] += 1
    res = {}
    cur = None
    for line in run("cuobjdump", "--dump-resource-usage", LIB).splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "REG:" in line:
            d = dict(kv.split(":") for kv in line.split() if ":" in kv)
            res[cur] = (int(d.get("REG", 0)), int(d.get("SHARED", 0)), int(d.get("LOCAL", 0)))
            cur = None
    names = demangle(sorted(counts))
    arch = re.search(r"arch = (\S+)", run("cuobjdump", "-lelf", LIB) + sass)
    print(f"# tools/sass_inventory.py over macaw-llm_b200/libmacaw_b200.so ({arch.group(1) if arch else '?'}; "
          f"{len(counts)} kernels; cuobjdump -sass / --dump-resource-usage, no GPU involved)")
    print("# HGMMA = wgmma.mma_async (HGMMA / QGMMA), UTMALDG = TMA tensor load, SYNCS = mbarrier operations, WARPGROUP = warpgroup")
    print("# arrive / wait, HMMA = mma.sync, LOCAL = spill bytes")
    hdr = f"{'kernel':64s} {'REG':>4s} {'SMEM':>6s} {'LOCAL':>5s} " + " ".join(f"{k:>12s}" for k in COLS)
    print(hdr)
    tot = defaultdict(int)
    for fnm in sorted(counts, key=lambda f: names[f]):
        reg, sh, loc = res.get(fnm, (0, 0, 0))
        c = counts[fnm]
        for k in COLS:
            tot[k] += c[k]
        print(f"{names[fnm][:64]:64s} {reg:4d} {sh:6d} {loc:5d} " + " ".join(f"{c[k]:12d}" for k in COLS))
    print(f"{'TOTAL':64s} {'':4s} {'':6s} {'':5s} " + " ".join(f"{tot[k]:12d}" for k in COLS))
    hm = [names[f] for f in counts if counts[f]["HMMA"]]
    print("# kernels containing HMMA (mma.sync): " + (", ".join(sorted(hm)) if hm else "none"))
    spill = [names[f] for f in counts if res.get(f, (0, 0, 0))[2]]
    print("# kernels with local-memory (spill) bytes: " + (", ".join(sorted(spill)) if spill else "none"))


if __name__ == "__main__":
    main()
