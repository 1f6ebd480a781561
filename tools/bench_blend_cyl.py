"""Cylinder mode's composite two ways, alternated in one process: (a) warp first — pano_cyl_warp_batch_rgb8_dev writes
every warped image as f32, then pano_blend_dev blends them — and (b) the cylinder blend stream
(pano_blend_stream_create_cyl), which reads the unwarped 8-bit sources and stores no warped image, with windows of 1
and of n images:

  python tools/bench_blend_cyl.py                  # config 1 shape, 13 × 1500×1112, 24 × 4000×3000; linear and 5 bands
  python tools/bench_blend_cyl.py --jobs config1 --bands 0

Sources are seeded random 8-bit RGB images on the device (the composite's cost does not depend on their content),
laid out as a horizontal strip at a fixed step, the way cylinder mode's ordered input is.  Per row: the median wall
time to the mosaic on the device (a host clock around the calls, ending in a stream synchronise), the per-kernel
times of one profiled run, and the context pool's high-water mark (PANO_CACHE_MB=0; it includes the 8-bit device
sources and the mosaic buffer, which both paths hold).  Every stream mosaic is checked bit for bit
against the warp-first one.  Prints the card's name and power limit with the numbers.  Needs an H100."""
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

JOBS = {   # name: (n, w, h, step)
    "config1": (8, 600, 400, 200),
    "13x1500x1112": (13, 1500, 1112, 500),
    "24x4000x3000": (24, 4000, 3000, 2000),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", default=",".join(JOBS))
    ap.add_argument("--bands", default="0,5")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    os.environ["PANO_CACHE_MB"] = "0"
    from openpano_b200 import synth
    from openpano_b200._abi import default_params
    from openpano_b200.capi import SRC_RGB8_DEV, Engine

    eng = Engine(0)
    print(json.dumps(dict(card=card())), flush=True)
    results = []
    for job in a.jobs.split(","):
        n, w, h, step = JOBS[job]
        rng = np.random.RandomState(n)
        pix = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for _ in range(n)]
        params = default_params(ordered_input=1)
        ow, oh, _, _ = eng.cyl_warp_shape(w, h, 1.0, params)
        items, geom = synth.translation_blend_setup([(k * step, 0) for k in range(n)], ow, oh)
        tw, th = max(it[2] for it in items), max(it[3] for it in items)
        d_pix = [eng.dev_alloc(p.nbytes) for p in pix]
        for d, p in zip(d_pix, pix):
            eng.dev_upload(d, p)
        del pix
        d_out = eng.dev_alloc(tw * th * 12)
        for bands in [int(b) for b in a.bands.split(",")]:
            def warp_first():
                d_warp = [eng.dev_alloc(ow * oh * 12) for _ in range(n)]
                eng.cyl_warp_batch_rgb8_dev(d_pix, [3] * n, [(h, w)] * n, d_warp, None, 1.0, params)
                eng.blend_dev(d_warp, [(oh, ow)] * n, items, geom, d_out, tw, th, bands, params)
                for d in d_warp:
                    eng.dev_free(d)

            def stream(win):
                def run():
                    s = eng.blend_stream_cyl([(h, w)] * n, items, geom, 1.0, bands, params)
                    try:
                        for k in range(0, n, win):
                            s.add(d_pix[k:k + win], SRC_RGB8_DEV)
                        s.finish_dev(d_out)
                    finally:
                        s.close()
                return run

            paths = {"warp then blend": warp_first, "stream w1": stream(1), f"stream w{n}": stream(n)}
            want = got = None
            wall = {k: [] for k in paths}
            mark = {k: 0 for k in paths}
            for fn in paths.values():                 # warm-up of every shape
                fn()
                eng.sync()
            for rep in range(a.reps):                  # alternated
                for name, fn in paths.items():
                    eng.sync()
                    eng.mem_high_water(reset=True)
                    t0 = time.perf_counter()
                    fn()
                    eng.sync()
                    wall[name].append((time.perf_counter() - t0) * 1e3)
                    mark[name] = max(mark[name], eng.mem_high_water())
                    if rep == 0:
                        out = np.empty((th, tw, 3), np.float32)
                        eng.dev_download(out, d_out)
                        if want is None:
                            want = out
                        else:
                            got = out
                            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{job} {name} differs"
            kernels = {}
            for name, fn in paths.items():             # per-kernel times: one profiled run each, apart
                eng.sync()
                eng.profile(True)
                eng.profile_reset()
                fn()
                eng.sync()
                kernels[name] = {k: round(v[1], 3) for k, v in sorted(eng.profile_read().items())}
                eng.profile(False)
            for name in paths:
                row = dict(job=job, n=n, src=[w, h], warped=[ow, oh], canvas=[tw, th], bands=bands, path=name,
                           wall_ms=round(statistics.median(wall[name]), 2),
                           wall_ms_spread=[round(min(wall[name]), 2), round(max(wall[name]), 2)],
                           mark_gb=round(mark[name] / 1e9, 3), kernels_ms=kernels[name])
                results.append(row)
                print(json.dumps(row), flush=True)
            del want, got
        for d in d_pix + [d_out]:
            eng.dev_free(d)
        eng.trim()
    print(json.dumps(dict(card=card(), rows=len(results))))
    eng.close()


if __name__ == "__main__":
    main()
