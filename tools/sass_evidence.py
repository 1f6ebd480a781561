#!/usr/bin/env python
"""Instruction counts that show the Hopper-native paths, per kernel, from the built library:
  python tools/sass_evidence.py > sass_evidence.txt"""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
so = sys.argv[1] if len(sys.argv) > 1 else str(ROOT / "openpano_b200" / "libpano_b200.so")
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
WATCH = re.compile(r"^(UTMALDG|UTMASTG|UTMACCTL|UBLKCP|HGMMA|WARPGROUP|SYNCS|FFMA|DFMA|DMUL|DADD|MUFU|HMMA|VIMNMX3?|FENCE)")
per = collections.OrderedDict()
cur = None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        cur = per.setdefault(name, collections.Counter())
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur is not None:
        op = m.group(1)
        if WATCH.match(op):
            key = op.rstrip(".") if op.startswith(("SYNCS", "HGMMA", "WARPGROUP", "UBLKCP", "UTMA")) else op.split(".")[0]
            cur[key] += 1
print("# SASS evidence (cuobjdump -sass openpano_b200/libpano_b200.so, sm_90a), instruction counts per kernel")
print("# wgmma.mma_async -> HGMMA; wgmma fence / wait -> WARPGROUP.*; cp.async.bulk.tensor -> UTMALDG; cp.async.bulk -> UBLKCP;")
print("# mbarrier -> SYNCS.*.  FFMA/DFMA that remain under --fmad=false sit inside the IEEE")
print("# division / square-root sequences (MUFU seed + FMA refinement), not in contracted multiply-adds.\n")
for name, c in per.items():
    if not c:
        continue
    if any(k.startswith(("UTMALDG", "HGMMA", "UBLKCP")) for k in c) or name.startswith(("k_descriptor", "k_linear_blend", "k_orientation")):
        print(f"{name}: " + ", ".join(f"{k} x{v}" for k, v in sorted(c.items(), key=lambda kv: -kv[1])))
