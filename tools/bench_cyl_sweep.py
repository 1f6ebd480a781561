"""Time, peak device memory and PCIe traffic of cylinder mode's output end, write_rgb(crop(CylinderStitcher::build())):
the cylinder sweep (`stitcher.cylinder_mosaic_rgb8_sweep`: each strip of the corrected canvas blends the band of
mosaic rows its perspective correction reads, from the unwarped sources) at strips of 256 and 1024 rows, against the
same chain over the whole canvas in one strip (the cylinder stream's whole f32 mosaic, the correction of every row,
crop, 8-bit conversion):

  python tools/bench_cyl_sweep.py                 # config 1 (8 × 600×400) linear; 24 × 4000×3000 at 0 and 5 bands
  python tools/bench_cyl_sweep.py --reps 5 --big-n 12

Every path starts from pinned host 8-bit sources and ends with the cropped 8-bit mosaic on the host.  The correction
is a mild keystone (the top edge 4 % narrower), as the h-factor search leaves it.  Each sweep runs at keep_bytes
unlimited and at the plan's largest kept set ("live").  All paths of one shape are warmed up once and then timed
alternately, `--reps` rounds; times are the median wall ms of the whole call, `mark` the context pool's high-water
mark during the call with PANO_CACHE_MB=0, `uploads_gb` the bytes that crossed PCIe (pano_blend_sweep_stats).  Every
output is checked byte for byte against the whole-canvas one.  The card's name and power limit are read in the same
run.  Needs an H100."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--big-n", type=int, default=24, help="images of the 4000×3000 stack (0: skip it)")
    ap.add_argument("--strips", default="256,1024")
    a = ap.parse_args()
    os.environ["PANO_CACHE_MB"] = "0"
    import torch
    from openpano_b200 import synth
    from openpano_b200._abi import default_params
    from openpano_b200.capi import SIZE_MAX, SRC_RGB8_HOST, Engine, blend_sweep_plan_cyl
    from openpano_b200.stitcher import cylinder_mosaic_rgb8_sweep
    from tests.persp_util import keystone

    eng = Engine(0)
    rows = []

    def measure(paths, reps):
        """{name: (median wall ms, pool high-water bytes, last result)}: every path warmed once, then timed in
        alternating rounds."""
        for _, fn in paths:
            fn()
        wall = {name: [] for name, _ in paths}
        mark = {name: 0 for name, _ in paths}
        out = {}
        for _ in range(reps):
            for name, fn in paths:
                eng.sync()
                eng.mem_high_water(reset=True)
                t0 = time.perf_counter()
                out[name] = fn()
                eng.sync()
                wall[name].append((time.perf_counter() - t0) * 1e3)
                mark[name] = max(mark[name], eng.mem_high_water())
        return {name: (statistics.median(wall[name]), mark[name], out[name]) for name, _ in paths}

    def record(**kw):
        rows.append(kw)
        print(json.dumps(kw), flush=True)

    def shape(label, stack, n, max_out, bands_list):
        imgs, org = synth.config_stack(stack, n)
        n, (h, w) = len(imgs), imgs[0].shape[:2]
        host = [torch.from_numpy((im * 255.0 + 0.5).astype(np.uint8)).pin_memory() for im in imgs]
        del imgs
        src = [t.data_ptr() for t in host]
        shapes = [(h, w)] * n
        nbytes = [h * w * 3] * n
        ow_w, oh_w, _, _ = Engine.cyl_warp_shape(w, h)
        items, geom = synth.translation_blend_setup(org, ow_w, oh_w, max_out)
        ow, oh = max(it[2] for it in items), max(it[3] for it in items)
        inv = keystone(ow, oh, 0.04, 0.0, 0.01)
        for bands in bands_list:
            p = default_params(multiband=bands, lazy_read=0)

            def sweep(strip, keep, stats):
                def run():
                    return cylinder_mosaic_rgb8_sweep(eng, items, geom, 1.0, inv, bands, src, strip, keep,
                                                      params=p, kind=SRC_RGB8_HOST, formats=[3] * n, shapes=shapes,
                                                      stats=stats)
                return run
            stats = {}
            paths = [("whole canvas (one strip)", sweep(oh, SIZE_MAX, stats.setdefault("whole", {})))]
            for strip in [int(x) for x in a.strips.split(",")]:
                pl = blend_sweep_plan_cyl(shapes, items, geom, bands, inv, strip, nbytes, SIZE_MAX, p)
                live = pl["retained_high"]
                band = int((pl["band"][:, 1] - pl["band"][:, 0]).max())
                for keep, kname in ((SIZE_MAX, "unlimited"), (live, f"live ({live / 1e9:.3f} GB)")):
                    name = f"sweep, strips of {strip} (tallest band {band}), keep={kname}"
                    paths.append((name, sweep(strip, keep, stats.setdefault(name, {}))))
            res = measure(paths, a.reps)
            want_rect, want = res["whole canvas (one strip)"][2]
            for name, (t, m, (rect, px)) in res.items():
                assert np.array_equal(rect, want_rect) and px.tobytes() == want.tobytes(), name
                st = stats["whole" if name.startswith("whole") else name]
                record(shape=label, bands=bands, row=name, wall_ms=round(t, 1), mark_gb=round(m / 1e9, 3),
                       uploads_gb=round(st["upload_bytes"] / 1e9, 3), canvas=[ow, oh])
        del host

    shape("config 1: 8 x 600x400", "cmu0_8x600x400", None, None, [0])
    if a.big_n:
        shape(f"{a.big_n} x 4000x3000", "uav_64x4000x3000", a.big_n, 8000, [0, 5])
    print(json.dumps(dict(gpu=card(), torch_device=torch.cuda.get_device_name(0), rows=rows)))
    eng.close()


if __name__ == "__main__":
    main()
