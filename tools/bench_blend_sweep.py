"""Time, peak device memory and PCIe traffic of the blend sweep (`stitcher.mosaic_rgb8_sweep`: each source uploaded
once while later strips read it, within keep_bytes) against the strip-by-strip writer (`mosaic_rgb8_strips`, one
upload per strip that reads a source) and the whole-canvas blend stream followed by pano_crop_rect_dev and
pano_mat32f_to_rgb8_dev, on config 5's blend stage (64 × 4000×3000, canvas 8000×6000):

  python tools/bench_blend_sweep.py                      # linear and 5 bands, strips of 256, 1024 and 4096 rows
  python tools/bench_blend_sweep.py --bands 0 --strips 256 --reps 3

Every path starts from pinned host 8-bit sources and ends with the cropped 8-bit mosaic on the host.  For each strip
height the sweep runs at keep_bytes 0, at the plan's largest kept set ("live": the least budget that uploads each
source once) and without a limit.  All paths of one strip height are warmed up once and then timed alternately,
`--reps` rounds; times are the median wall ms of the whole call, `mark` the context pool's high-water mark during
the call with PANO_CACHE_MB=0, `uploads_gb` the bytes that crossed PCIe (pano_blend_sweep_stats for the sweep, the
read sets for the strips).  Every output is checked byte for byte against the whole-canvas one.  The card's name
and power limit are read in the same run.  Needs an H100."""
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
    ap.add_argument("--n", type=int, default=64, help="images of config 5's stack")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--bands", default="0,5")
    ap.add_argument("--strips", default="256,1024,4096")
    a = ap.parse_args()
    os.environ["PANO_CACHE_MB"] = "0"
    import torch
    from openpano_b200 import synth
    from openpano_b200._abi import default_params
    from openpano_b200.capi import SIZE_MAX, SRC_RGB8_HOST, Engine, blend_sweep_plan
    from openpano_b200.stitcher import mosaic_rgb8_strips, mosaic_rgb8_sweep

    imgs, org = synth.config_stack("uav_64x4000x3000", a.n)
    n, (h, w) = len(imgs), imgs[0].shape[:2]
    host = [torch.from_numpy((im * 255.0 + 0.5).astype(np.uint8)).pin_memory() for im in imgs]
    del imgs
    src = [t.data_ptr() for t in host]
    shapes = [(h, w)] * n
    nbytes = [h * w * 3] * n
    items, geom = synth.translation_blend_setup(org, w, h, 8000)
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
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
                return rect, px.reshape(int(rect[3]), int(rect[2]), 3)
            finally:
                s.close()
                for d in (d_mos, d_rect, d_out):
                    eng.dev_free(d)
        return run

    for bands in [int(b) for b in a.bands.split(",")]:
        p = default_params(multiband=bands, lazy_read=0)
        res = measure([("whole", whole(bands, p))], a.reps)
        t, m, (want_rect, want) = res["whole"]
        record(bands=bands, row="whole canvas", wall_ms=round(t, 1), mark_gb=round(m / 1e9, 3),
               uploads_gb=round(sum(nbytes) / 1e9, 3))
        for strip in [int(x) for x in a.strips.split(",")]:
            none = blend_sweep_plan(shapes, items, geom, bands, strip, nbytes, 0)
            live = blend_sweep_plan(shapes, items, geom, bands, strip, nbytes, SIZE_MAX)["retained_high"]
            stats = {}

            def strips(strip=strip):
                return mosaic_rgb8_strips(eng, items, geom, bands, src, strip, 1, params=p, kind=SRC_RGB8_HOST,
                                          channels=3, shapes=shapes)

            def sweep(keep, strip=strip):
                def run():
                    st = stats.setdefault(keep, {})
                    return mosaic_rgb8_sweep(eng, items, geom, bands, src, strip, keep, params=p, kind=SRC_RGB8_HOST,
                                             formats=[3] * n, shapes=shapes, stats=st)
                return run
            paths = [("strips", strips)] + [(f"sweep keep={k}", sweep(k)) for k in (0, live, SIZE_MAX)]
            res = measure(paths, a.reps)
            for name, (t, m, (rect, px)) in res.items():
                assert np.array_equal(rect, want_rect) and px.tobytes() == want.tobytes(), f"{name}, strips of {strip}"
                if name == "strips":
                    up = none["upload_bytes"]
                else:
                    keep = int(name.split("=")[1])
                    up = stats[keep]["upload_bytes"]
                    name = "sweep keep=" + ("0" if keep == 0 else "unlimited" if keep == SIZE_MAX else
                                            f"live ({keep / 1e9:.3f} GB)")
                record(bands=bands, row=f"{name}, strips of {strip}", wall_ms=round(t, 1), mark_gb=round(m / 1e9, 3),
                       uploads_gb=round(up / 1e9, 3))
    print(json.dumps(dict(gpu=card(), torch_device=torch.cuda.get_device_name(0), n=n, w=w, h=h, canvas=[ow, oh],
                          rows=rows)))
    eng.close()


if __name__ == "__main__":
    main()
