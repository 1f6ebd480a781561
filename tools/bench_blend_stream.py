"""Device time and peak device memory of the windowed blend (pano_blend_stream_*) against the resident path
(every source on the device as f32, then pano_blend_dev), on a BASELINE config's blend stage:

  python tools/bench_blend_stream.py --config 5     # 64 × 4000×3000, MULTIBAND 5, MAX_OUTPUT_SIZE 8000
  python tools/bench_blend_stream.py --config 2     # 13 × 1500×1112 ordered, linear

Rows: `resident` (pano_blend_dev over f32 sources converted on the device from the 8-bit ones), `stream dev u8 wK`
(8-bit device sources, windows of K), `stream pinned u8 wK` (8-bit pinned host sources through the stream's two-slot
ring: wall time, H2D included) and `h2d only` (the same bytes uploaded on their own).  `mark` is the context pool's
high-water mark during the call with PANO_CACHE_MB=0; device-source rows include the 8-bit sources themselves.
Every stream output is checked bit for bit against the resident one.  Needs an H100."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import numpy as np  # noqa: E402

CONFIGS = {
    "5": dict(stack="uav_64x4000x3000", bands=5, params=dict(multiband=5, lazy_read=0), max_output=8000),
    "2": dict(stack="ordered_13x1500x1112", bands=0, params=dict(ordered_input=1), max_output=None),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=sorted(CONFIGS), default="5")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--windows", default="1,4,16")
    a = ap.parse_args()
    os.environ["PANO_CACHE_MB"] = "0"
    import torch
    from openpano_b200 import synth
    from openpano_b200._abi import default_params
    from openpano_b200.capi import SRC_RGB8_DEV, SRC_RGB8_HOST, Engine

    cfg = CONFIGS[a.config]
    imgs, org = synth.config_stack(cfg["stack"])
    n, (h, w) = len(imgs), imgs[0].shape[:2]
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    del imgs
    items, geom = synth.translation_blend_setup(org, w, h, cfg["max_output"])
    params, bands = default_params(**cfg["params"]), cfg["bands"]
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    shapes = [(h, w)] * n
    stream = torch.cuda.Stream()
    eng = Engine(0, stream=stream.cuda_stream)
    gpu = torch.cuda.get_device_name(0)
    rows = []

    def timed(fn):
        """(median device ms, median wall ms, pool high-water bytes) over reps, after one warm-up."""
        fn()
        eng.sync()
        dev, wall, mark = [], [], 0
        for _ in range(a.reps):
            eng.sync()
            eng.mem_high_water(reset=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(stream)
            fn()
            e1.record(stream)
            eng.sync()
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(e0.elapsed_time(e1))
            mark = max(mark, eng.mem_high_water())
        return statistics.median(dev), statistics.median(wall), mark

    def record(name, dev_ms, wall_ms, mark):
        rows.append(dict(row=name, device_ms=round(dev_ms, 2), wall_ms=round(wall_ms, 2), mark_gb=round(mark / 1e9, 3)))
        print(json.dumps(rows[-1]), flush=True)

    nb = h * w * 3
    d_pix = [eng.dev_alloc(nb) for _ in range(n)]
    for d, p in zip(d_pix, pix):
        eng.dev_upload(d, p)
    d_out = eng.dev_alloc(ow * oh * 12)
    want = np.empty((oh, ow, 3), np.float32)
    got = np.empty_like(want)

    def resident():
        d_f32 = [eng.dev_alloc(nb * 4) for _ in range(n)]
        eng.rgb8_to_mat32f_batch_dev(d_pix, [w] * n, [h] * n, [3] * n, d_f32)
        eng.blend_dev(d_f32, shapes, items, geom, d_out, ow, oh, bands, params)
        for d in d_f32:
            eng.dev_free(d)

    record("resident f32 (u8 convert + pano_blend_dev)", *timed(resident))
    eng.dev_download(want, d_out)

    def stream_run(ptrs, kind, win):
        def run():
            s = eng.blend_stream(shapes, items, geom, bands, params)
            try:
                for k in range(0, n, win):
                    s.add(ptrs[k:k + win], kind)
                s.finish_dev(d_out)
            finally:
                s.close()
        return run

    windows = [int(x) for x in a.windows.split(",")]
    for win in windows:
        record(f"stream dev u8 w{win}", *timed(stream_run(d_pix, SRC_RGB8_DEV, win)))
        eng.dev_download(got, d_out)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"dev u8 window {win} differs"
    for d in d_pix:
        eng.dev_free(d)
    host = [torch.from_numpy(p).pin_memory() for p in pix]
    hptr = [t.data_ptr() for t in host]
    for win in windows:
        record(f"stream pinned u8 w{win}", *timed(stream_run(hptr, SRC_RGB8_HOST, win)))
        eng.dev_download(got, d_out)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"pinned u8 window {win} differs"
    d_all = eng.dev_alloc(nb * n)

    def h2d():
        for k, p in enumerate(hptr):
            eng.dev_upload_async(d_all + k * nb, p, nb)

    record("h2d only (all 8-bit sources, pinned)", *timed(h2d))
    eng.dev_free(d_all)
    eng.dev_free(d_out)
    print(json.dumps(dict(config=a.config, gpu=gpu, n=n, w=w, h=h, canvas=[ow, oh], bands=bands,
                          u8_source_gb=round(nb * n / 1e9, 3), f32_source_gb=round(4 * nb * n / 1e9, 3), rows=rows)))
    eng.close()


if __name__ == "__main__":
    main()
