"""Time and peak device memory of the windowed SIFT (pano_sift_stream_*) against the batch
(pano_sift_detect_batch_rgb8), both from host 8-bit pixels, on config 5's shape (64 × 4000×3000):

  python tools/bench_sift_stream.py                    # windows of 1, 2, 4, 8 and 16
  python tools/bench_sift_stream.py --windows 4,64 --reps 5

Rows: `batch` (every source uploaded, then one SIFT batch), `stream wK` (windows of K through the stream's two-slot
ring), each from pageable numpy buffers (what a decoder hands over: staged through pinned memory on the host) and
from pinned ones.  Two rows show what the stream could at best overlap: `sift only` (one batch from device
sources, no upload) and `h2d only` (the pinned 8-bit sources uploaded on their own).  Times are wall ms from the
first call until the counts are on the host (one count query), median over reps after one warm-up; `mark` is the
context pool's high-water mark during the call with PANO_CACHE_MB=0.  Every stream featureset is checked bit for
bit against the batch's.  The card's name and power limit are read in the same run.  Needs an H100."""
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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--windows", default="1,2,4,8,16")
    a = ap.parse_args()
    os.environ["PANO_CACHE_MB"] = "0"
    import torch
    from openpano_b200 import synth
    from openpano_b200.capi import SRC_RGB8_HOST, Engine

    imgs, _ = synth.config_stack("uav_64x4000x3000", a.n)
    n, (h, w) = len(imgs), imgs[0].shape[:2]
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    del imgs
    nb = h * w * 3
    eng = Engine(0)
    rows = []

    def timed(fn):
        """(median wall ms, pool high-water bytes, the last featureset) over reps, after one warm-up."""
        fn().free()
        wall, mark, fs = [], 0, None
        for _ in range(a.reps):
            if fs is not None:
                fs.free()
            eng.sync()
            eng.mem_high_water(reset=True)
            t0 = time.perf_counter()
            fs = fn()
            fs.count(0)
            eng.sync()
            wall.append((time.perf_counter() - t0) * 1e3)
            mark = max(mark, eng.mem_high_water())
        return statistics.median(wall), mark, fs

    def record(name, wall_ms, mark, fs=None, want=None):
        if want is not None:
            for i in range(n):
                gc, gd = fs.download(i)
                wc, wd = want.download(i)
                assert gc.tobytes() == wc.tobytes() and gd.tobytes() == wd.tobytes(), f"{name}: image {i} differs"
        rows.append(dict(row=name, wall_ms=round(wall_ms, 1), mark_gb=round(mark / 1e9, 3)))
        print(json.dumps(rows[-1]), flush=True)

    def batch(src):
        return lambda: eng.sift_detect_batch_rgb8_ptr(src, [w] * n, [h] * n, [3] * n)

    def stream(src, win):
        def run():
            s = eng.sift_stream([(h, w)] * n)
            try:
                for k in range(0, n, win):
                    s.add(src[k:k + win], SRC_RGB8_HOST, 3)
                return s.finish()
            finally:
                s.close()
        return run

    windows = [int(x) for x in a.windows.split(",")]
    host = [torch.from_numpy(p).pin_memory() for p in pix]
    for label, src in (("pageable", [p.ctypes.data for p in pix]), ("pinned", [t.data_ptr() for t in host])):
        t, m, want = timed(batch(src))
        record(f"batch {label}", t, m)
        for win in windows:
            t, m, fs = timed(stream(src, win))
            record(f"stream {label} w{win}", t, m, fs, want)
            fs.free()
        want.free()

    d_all = eng.dev_alloc(nb * n)
    hptr = [t.data_ptr() for t in host]

    def h2d():
        t0 = time.perf_counter()
        for k, p in enumerate(hptr):
            eng.dev_upload_async(d_all + k * nb, p, nb)
        eng.sync()
        return (time.perf_counter() - t0) * 1e3

    h2d()
    record("h2d only (all 8-bit sources, pinned)", statistics.median([h2d() for _ in range(a.reps)]), 0)
    d_src = [d_all + k * nb for k in range(n)]
    t, m, fs = timed(lambda: eng.sift_detect_batch_rgb8_ptr(d_src, [w] * n, [h] * n, [3] * n, device=True))
    fs.free()
    record("sift only (batch from device sources)", t, m)
    eng.dev_free(d_all)
    print(json.dumps(dict(gpu=card(), torch_device=torch.cuda.get_device_name(0), n=n, w=w, h=h,
                          u8_source_gb=round(nb * n / 1e9, 3), rows=rows)))
    eng.close()


if __name__ == "__main__":
    main()
