"""Disassemble bodo_b200/libbodo_b200.so (cuobjdump -sass) and list, per kernel, the instructions that prove which hardware
paths it uses: UBLKCP (TMA bulk copy, cp.async.bulk), SYNCS (mbarrier), REDUX (warp reduce), ATOMS / ATOMG / RED (shared /
global atomics), LDG.E.128 / STG.E.128 (16-byte global accesses), plus the register count.  Output: stdout

    python benchmarks/sass_excerpt.py > sass_excerpt.txt
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bodo_b200", "libbodo_b200.so")
PATTERNS = ["UBLKCP", "SYNCS", "REDUX", "ATOMS", "ATOMG", "RED.", "LDG.E.128", "STG.E.128", "LDG.E.64", "STG.E.64", "LDS.128", "STS.128",
            "BAR.SYNC", "MATCH", "SHFL", "VOTE", "CCTL", "ERRBAR", "MEMBAR", "UTMALDG", "UTMASTG"]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    regs = {}
    cur = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        m = re.search(r"REG:(\d+)", line)
        if m and cur:
            regs[cur] = int(m.group(1))
    demangle = {}
    names = sorted(regs)
    if names:
        out = subprocess.run(["c++filt"] + names, capture_output=True, text=True).stdout.splitlines()
        demangle = dict(zip(names, out))
    counts = collections.OrderedDict()
    first = {}
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            first[cur] = {}
            continue
        if cur is None or "/*" not in line:
            continue
        m = re.search(r"/\*[0-9a-f]+\*/\s+(.*?);", line)
        if not m:
            continue
        ins = m.group(1).strip()
        counts[cur]["_total"] += 1
        for p in PATTERNS:
            if p in ins.split()[0] or (ins.startswith("@") and len(ins.split()) > 1 and p in ins.split()[1]):
                counts[cur][p] += 1
                first[cur].setdefault(p, ins)
    print(f"# SASS excerpt of {os.path.relpath(LIB, ROOT)} (cuobjdump -sass, sm_90a only); counts are static instruction sites")
    arch = set(re.findall(r"arch = (sm_\w+)", sass))
    print(f"# architectures in the fatbin: {sorted(arch)}")
    for fn, c in counts.items():
        name = demangle.get(fn, fn)
        name = re.sub(r"b200::", "", name)
        tags = ", ".join(f"{p} x{c[p]}" for p in PATTERNS if c[p])
        print(f"\n{name}\n    regs {regs.get(fn, '?')}, {c['_total']} SASS instructions; {tags or 'no listed instruction classes'}")
        for p in ("UBLKCP", "SYNCS", "REDUX", "ATOMS", "RED.", "ATOMG", "STG.E.128"):
            if p in first[fn]:
                print(f"        e.g. {first[fn][p]}")


if __name__ == "__main__":
    sys.exit(main())
