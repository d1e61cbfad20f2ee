#!/usr/bin/env python
"""Per-kernel opcode histogram of the product library's SASS (cuobjdump -sass) with its resource usage.

    python tools/sass_table.py [lib.so] > profiles/r2_sass_opcodes.txt
Shows, kernel by kernel, which memory / shuffle / tensor / bulk-copy instructions the compiler emitted
(e.g. LDG.E.128.CONSTANT = the read-only point loads, DMMA = the fp64 tensor-core fold of the fit kernel).
"""
import collections, re, subprocess, sys
lib = sys.argv[1] if len(sys.argv) > 1 else "limo-velo_b200/liblimovelo_b200.so"
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
res = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True).stdout
usage = {}
cur = None
for l in res.splitlines():
    m = re.match(r"\s*Function (\S+):", l)
    if m: cur = m.group(1); continue
    if cur and "REG:" in l: usage[cur] = l.strip(); cur = None
demangle = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
kern, ops = None, None
out = []
def flush():
    if kern and ops is not None and ("lv" in kern and "cub" not in kern):
        out.append((kern, ops))
for l in sass.splitlines():
    m = re.match(r"\s*Function : (\S+)", l)
    if m:
        flush(); kern, ops = m.group(1), collections.Counter(); continue
    m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", l)
    if m and ops is not None: ops[m.group(1)] += 1
flush()
KEEP = re.compile(r"^(LDG|STG|LDS|STS|LDL|STL|LDC|ATOM|ATOMG|ATOMS|RED|SHFL|VOTE|MATCH|BAR|SYNCS|UBLKCP|UTMA|ACQBULK|FENCE|MEMBAR|ERRBAR|CCTL|DFMA|DADD|DMUL|DSETP|MUFU|FLO|POPC|BREV|HMMA|DMMA|IMMA|UTCMMA|TCGEN|WARPSYNC|NANOSLEEP|LDGDEPBAR|DEPBAR|ACQ|PREEXIT|S2UR)")
for k, o in sorted(out, key=lambda t: -sum(t[1].values())):
    print(demangle(k))
    print("   ", usage.get(k, ""), " | SASS instructions:", sum(o.values()))
    groups = collections.Counter()
    for op, n in o.items():
        if KEEP.match(op): groups[op] += n
    line = ", ".join(f"{op} x{n}" for op, n in sorted(groups.items()))
    while line:
        print("    " + line[:150]); line = line[150:]
    print()
