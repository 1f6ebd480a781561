#!/usr/bin/env python
"""Profiling target: N full steps of the bench workload on ONE context — 8-bit pixels
-> Mat32f, SIFT, match, linear blend, crop, 8-bit mosaic — so that ncu sees every
kernel of the path once per step.

  ncu --set full --import-source on --clock-control none --launch-skip <launches of step 0> \\
      -o out/prof python tools/one_step.py 2
"""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
from openpano_b200.capi import Engine  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 2
imgs, pairs, items, geom, params, mpx, pix = bench.make_workload(0, 0)
shapes = [im.shape[:2] for im in imgs]
ow, oh = max(it[2] for it in items), max(it[3] for it in items)
eng = Engine(0)
d_pix = [eng.dev_alloc(p.nbytes + 256) for p in pix]
d_img = [eng.dev_alloc(im.nbytes) for im in imgs]
d_out = eng.dev_alloc(ow * oh * 12)
d_out8 = eng.dev_alloc(ow * oh * 3 + 256)
for d, p in zip(d_pix, pix):
    eng.dev_upload(d, p)
ws, hs = [s[1] for s in shapes], [s[0] for s in shapes]
for step in range(steps):
    l0 = eng.launch_count()
    eng.rgb8_to_mat32f_batch_dev(d_pix, ws, hs, [3] * len(pix), d_img)
    fs = eng.sift_detect_batch_ptr(d_img, ws, hs, params, device=True)
    n = eng.match_pairs_dev(fs, pairs, params)
    eng.blend_dev(d_img, shapes, items, geom, d_out, ow, oh, 0, params)
    eng.crop_rect_dev(d_out, ow, oh, d_out8)
    eng.mat32f_to_rgb8_dev(d_out, ow, oh, d_out8, d_out8 + 256)
    eng.sync()
    fs.free()
    print(f"step {step}: {eng.launch_count() - l0} launches, {n} matches", flush=True)
eng.close()
