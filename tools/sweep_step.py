#!/usr/bin/env python
"""Profiling target: the brute-force match of the config-4 sweep at one size, N times.
  ncu --set full -k regex:k_tc_pass --launch-skip 7 -c 2 -o out/sweep python tools/sweep_step.py 100000 2
(a match call launches k_tc_pass seven times with columns on demand — first pass, then nomination and
filter in each of three rounds — so skip 7 lands on the second call's first pass and nomination)
"""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from openpano_b200._abi import default_params  # noqa: E402
from openpano_b200.capi import Engine  # noqa: E402
from tools.bench_configs import sweep_sets  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
a, b = sweep_sets(n)
eng = Engine(0)
fs = eng.featureset_upload([a, b])
for step in range(steps):
    tot = eng.match_pairs_dev(fs, [(0, 1)], default_params())
    print(f"step {step}: {tot} matches", flush=True)
fs.free()
