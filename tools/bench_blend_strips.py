"""Time and peak device memory of the 8-bit mosaic built strip by strip (row-strip blend streams, the crop scan
and the 8-bit crop: `stitcher.mosaic_rgb8_strips`) against the whole-canvas blend stream followed by
pano_crop_rect_dev and pano_mat32f_to_rgb8_dev, on config 5's blend stage (64 × 4000×3000, canvas 8000×6000):

  python tools/bench_blend_strips.py                     # linear and 5 bands, strips of 256, 1024 and 4096 rows
  python tools/bench_blend_strips.py --bands 0 --strips 512 --reps 3

Every path starts from pinned host 8-bit sources added one per window and ends with the cropped 8-bit mosaic on
the host.  Times are wall ms of the whole call, median over reps after one warm-up; `mark` is the context pool's
high-water mark during the call with PANO_CACHE_MB=0.  A strip stream uploads every image it needs, so an image
that reaches k strips is uploaded k times: `uploads_gb` counts those bytes.  Every strip output is checked byte
for byte against the whole-canvas one.  One more row runs a synthetic linear canvas wider than 40,000 columns,
which pano_crop_rect_dev refuses, through strips of 1024 rows.  For strips of 1024 rows of config 5 (linear) and
of the wide canvas, one more profiled run gives the device ms and launches of the crop scan's kernels (`crop_ms`):
k_crop_line, the line kernel in shared memory up to 40,000 columns, and k_crop_scan_line, which reads the heights
from global memory beyond.  The card's name and power limit are read in the same run.  Needs an H100."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import numpy as np  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def halo(bands):
    """Summed blur half-widths at GAUSS_WINDOW_FACTOR 6 (include/pano_b200.h)."""
    return {0: 0, 1: 0, 2: 6, 3: 12, 4: 18, 5: 27}[bands]


def uploads(items, bands, oh, strip, nbytes):
    """Bytes a strip run uploads: each image once per strip that needs it (pano_blend_stream_needs' rule)."""
    total = 0
    for r0 in range(0, oh, strip):
        r1 = min(oh, r0 + strip)
        if r0 == 0 and r1 == oh:
            total += nbytes * len(items)
            continue
        H = halo(bands)
        for _, y0, _, y1, _ in items:
            if bands == 0:
                total += nbytes * (y0 < r1 and y1 >= r0)
            else:
                c0 = max(0, r0 - H) if r0 > 0 else y0
                c1 = r1 + H - 1 if r1 < oh else y1
                total += nbytes * (max(y0, c0) <= min(y1, c1))
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64, help="images of config 5's stack")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--bands", default="0,5")
    ap.add_argument("--strips", default="256,1024,4096")
    a = ap.parse_args()
    os.environ["PANO_CACHE_MB"] = "0"
    import torch
    from openpano_b200 import synth
    from openpano_b200._abi import default_params
    from openpano_b200.capi import SRC_RGB8_HOST, Engine
    from openpano_b200.stitcher import mosaic_rgb8_strips

    imgs, org = synth.config_stack("uav_64x4000x3000", a.n)
    n, (h, w) = len(imgs), imgs[0].shape[:2]
    host = [torch.from_numpy((im * 255.0 + 0.5).astype(np.uint8)).pin_memory() for im in imgs]
    del imgs
    src = [t.data_ptr() for t in host]
    shapes = [(h, w)] * n
    items, geom = synth.translation_blend_setup(org, w, h, 8000)
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    eng = Engine(0)
    rows = []

    def timed(fn):
        """(median wall ms, pool high-water bytes, the last result) over reps, after one warm-up."""
        fn()
        wall, mark, out = [], 0, None
        for _ in range(a.reps):
            eng.sync()
            eng.mem_high_water(reset=True)
            t0 = time.perf_counter()
            out = fn()
            eng.sync()
            wall.append((time.perf_counter() - t0) * 1e3)
            mark = max(mark, eng.mem_high_water())
        return statistics.median(wall), mark, out

    def crop_profile(fn):
        """device ms and launches of the crop kernels in one profiled run of fn"""
        eng.profile(True)
        eng.profile_reset()
        fn()
        eng.sync()
        prof = eng.profile_read()
        eng.profile(False)
        return {k: dict(launches=v[0], ms=round(v[1], 3)) for k, v in prof.items() if k.startswith("k_crop")}

    def record(**kw):
        rows.append(kw)
        print(json.dumps(kw), flush=True)

    def whole(bands, p):
        def run():
            d_mos, d_rect, d_out = eng.dev_alloc(ow * oh * 12), eng.dev_alloc(256), eng.dev_alloc(ow * oh * 3)
            s = eng.blend_stream(shapes, items, geom, bands, p)
            try:
                for k in range(n):
                    s.add(src[k:k + 1], SRC_RGB8_HOST, 3)
                s.finish_dev(d_mos)
                eng.crop_rect_dev(d_mos, ow, oh, d_rect)
                eng.mat32f_to_rgb8_dev(d_mos, ow, oh, d_rect, d_out)
                rect = np.zeros(4, np.int32)
                eng.dev_download(rect, d_rect)
                px = np.empty(int(rect[2]) * int(rect[3]) * 3, np.uint8)
                eng.dev_download(px, d_out)
                return rect, px
            finally:
                s.close()
                for d in (d_mos, d_rect, d_out):
                    eng.dev_free(d)
        return run

    for bands in [int(b) for b in a.bands.split(",")]:
        p = default_params(multiband=bands, lazy_read=0)
        t, m, (want_rect, want) = timed(whole(bands, p))
        record(bands=bands, row="whole canvas", wall_ms=round(t, 1), mark_gb=round(m / 1e9, 3),
               uploads_gb=round(n * h * w * 3 / 1e9, 3))
        for strip in [int(x) for x in a.strips.split(",")]:

            def run(strip=strip):
                return mosaic_rgb8_strips(eng, items, geom, bands, src, strip, 1, params=p, kind=SRC_RGB8_HOST,
                                          channels=3, shapes=shapes)
            t, m, (rect, px) = timed(run)
            assert np.array_equal(rect, want_rect) and px.tobytes() == want.tobytes(), f"strips of {strip} differ"
            extra = dict(crop_ms=crop_profile(run)) if bands == 0 and strip == 1024 else {}
            record(bands=bands, row=f"strips of {strip}", wall_ms=round(t, 1), mark_gb=round(m / 1e9, 3),
                   uploads_gb=round(uploads(items, bands, oh, strip, h * w * 3) / 1e9, 3), **extra)

    # a synthetic canvas wider than pano_crop_rect_dev's 40,000 columns: 48 images of 2000×1000, 1000 columns apart
    wi, hi, nw = 2000, 1000, 48
    wimgs, worg = synth.make_stack(nw, wi, hi, 1000, 71)
    worg = [(x, y + (k * 37) % 200) for k, (x, y) in enumerate(worg)]
    wpix = [(im * 255.0 + 0.5).astype(np.uint8) for im in wimgs]
    del wimgs
    witems, wgeom = synth.translation_blend_setup(worg, wi, hi)
    wow, woh = max(it[2] for it in witems), max(it[3] for it in witems)

    def wide():
        return mosaic_rgb8_strips(eng, witems, wgeom, 0, wpix, 1024, 1)
    t, m, (rect, _) = timed(wide)
    record(bands=0, row=f"wide canvas {wow}x{woh}, strips of 1024", wall_ms=round(t, 1), mark_gb=round(m / 1e9, 3),
           rect=[int(v) for v in rect], crop_ms=crop_profile(wide))
    print(json.dumps(dict(gpu=card(), torch_device=torch.cuda.get_device_name(0), n=n, w=w, h=h, canvas=[ow, oh],
                          rows=rows)))
    eng.close()


if __name__ == "__main__":
    main()
