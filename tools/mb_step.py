#!/usr/bin/env python
"""Profiling target: the 5-band MultiBandBlender on the 13x1500x1112 stack, N times.
  ncu --set full -k regex:k_mb --launch-skip 12 -c 12 -o out/mb python tools/mb_step.py 2
"""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from openpano_b200 import synth  # noqa: E402
from openpano_b200._abi import default_params  # noqa: E402
from openpano_b200.capi import Engine  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 2
bands = int(sys.argv[2]) if len(sys.argv) > 2 else 5
imgs, org = synth.config_stack("ordered_13x1500x1112")
items, geom = synth.translation_blend_setup(org, 1500, 1112)
params = default_params(ordered_input=1, multiband=bands)
shapes = [im.shape[:2] for im in imgs]
ow, oh = max(it[2] for it in items), max(it[3] for it in items)
eng = Engine(0)
d_img = [eng.dev_alloc(im.nbytes) for im in imgs]
for d, im in zip(d_img, imgs):
    eng.dev_upload(d, im)
d_out = eng.dev_alloc(ow * oh * 12)
for step in range(steps):
    l0 = eng.launch_count()
    eng.blend_dev(d_img, shapes, items, geom, d_out, ow, oh, bands, params)
    eng.sync()
    print(f"step {step}: {eng.launch_count() - l0} launches", flush=True)
