#!/usr/bin/env python
"""Opcode histogram per kernel of the built library (cuobjdump -sass): instruction count, the Hopper bulk-copy
mnemonics (UBLKCP = cp.async.bulk, SYNCS = mbarrier), stores by
width, and the 25 most frequent opcodes.  usage: sass_histogram.py [lib.so] > profiles/rNN/sass_histogram.txt"""
import collections, re, subprocess, sys
lib = sys.argv[1] if len(sys.argv) > 1 else "gofr_b200/libgofr_b200.so"
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
fn, per = None, collections.OrderedDict()
for ln in out.splitlines():
    m = re.search(r"Function : (\S+)", ln)
    if m:
        fn = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        per[fn] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln)
    if m and fn:
        per[fn][m.group(1)] += 1
arch = re.search(r"arch = (sm_\w+)", out)
print(f"{lib}: {arch.group(1) if arch else '?'} cubins\n")
for fn, c in per.items():
    total = sum(c.values())
    def grp(pred):
        return sum(v for k, v in c.items() if pred(k))
    print(f"== {fn}: {total} instructions ({total * 16 / 1024:.1f} KB)")
    print(f"   bulk copy / mbarrier: UBLKCP {grp(lambda k: k.startswith('UBLKCP'))}, SYNCS {grp(lambda k: k.startswith('SYNCS'))};"
          f" tensor-core / TMEM ops: {grp(lambda k: k.startswith('UTC') or k.startswith('LDTM') or k.startswith('STTM') or 'MMA' in k)} (byte path: none expected)")
    print(f"   global stores: 256-bit {grp(lambda k: k.startswith('STG') and '.256' in k)}, 128-bit {grp(lambda k: k.startswith('STG') and '.128' in k)},"
          f" narrower {grp(lambda k: (k.startswith('STG') or k.startswith('ST.E')) and '.128' not in k and '.256' not in k)};"
          f" shared: LDS {grp(lambda k: k.startswith('LDS'))}, STS {grp(lambda k: k.startswith('STS'))}; local: LDL {grp(lambda k: k.startswith('LDL'))}, STL {grp(lambda k: k.startswith('STL'))}")
    base = collections.Counter()
    for k, v in c.items():
        base[k.split(".")[0]] += v
    print("   top opcodes: " + ", ".join(f"{k} {v}" for k, v in base.most_common(25)) + "\n")
