#!/usr/bin/env python
"""Cost of the little-planet view from a decoded 8-bit image (pano_planet_pix8[_dev]) against the f32 entry point
(pano_planet[_dev]) on read_img's image of the same pixels.  One JSON line:

  device         card name and power limit, read by one nvidia-smi call in this run
  shapes         the CMU1 mosaic of the reference's run_test.py (8000×1449) and config 5's 8000×6000 canvas, the
                 largest cropped mosaic config 5 can give
  wall_ms        per shape and input: host wall time of one call from host pixels to the planet on the host (upload,
                 kernel, 12 MB download, stream sync), median of --wall-iters calls after --warmup, from pageable
                 (numpy) and pinned (pano_host_alloc) buffers; the input is each PANO_PIX_* format for
                 pano_planet_pix8 and read_img's f32 image for pano_planet
  kernel_ms      per shape: device time of each kernel instantiation between CUDA events on the engine's stream
                 (k_planet_rgb8 for grey and RGB, k_planet_pix8 for RGBA and planar, k_planet for f32), median (min,
                 max) of --iters launches after --warmup
  model_bytes    per shape and input: bytes uploaded (1, 3, 4 or 12 per input pixel), and per launch 16 B of table and
                 12 B of output per output pixel plus 4 taps of 1, 3, 4 or 12 B per coloured pixel (an upper bound on
                 the gathers: neighbouring pixels share taps), with the rate the kernel's median implies
Every planet is checked bit for bit against pano_planet on read_img's image before it is timed.  Needs an H100.

    python tools/bench_planet_pix8.py [--iters 200] [--warmup 10] [--wall-iters 10] [--out results/planet_pix8.jsonl]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from openpano_b200.capi import Engine  # noqa: E402
from tests import pix_util as xu  # noqa: E402

SHAPES = {"cmu1_8000x1449": (8000, 1449), "config5_canvas_8000x6000": (8000, 6000)}
FORMATS = {"grey": 1, "rgb": 3, "rgba": 4, "planar": 3}          # bytes per pixel
KERNEL = {"grey": "k_planet_rgb8", "rgb": "k_planet_rgb8", "rgba": "k_planet_pix8", "planar": "k_planet_pix8",
          "f32": "k_planet"}
OUT_PIXELS = Engine.PLANET_SIZE ** 2


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30)
    except FileNotFoundError:
        out = None
    if out is None or out.returncode != 0 or not out.stdout.strip():
        raise SystemExit("bench_planet_pix8: nvidia-smi found no GPU")
    name, power, clock = [x.strip() for x in out.stdout.strip().split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def layout(rgb, fmt):
    if fmt == "rgba":
        return xu.to_rgba(rgb, alpha_seed=1)
    if fmt == "planar":
        return xu.to_planar(rgb)
    if fmt == "grey":
        return np.ascontiguousarray(rgb[..., 0])
    return rgb


def pinned_copy(arr):
    """(pinned numpy array with arr's contents, pointer to free)"""
    ptr = Engine.host_alloc(arr.nbytes)
    view = np.ctypeslib.as_array((C.c_uint8 * arr.nbytes).from_address(ptr)).view(arr.dtype).reshape(arr.shape)
    view[...] = arr
    return view, ptr


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return round(float(np.median(t)) * 1e3, 3)


def kernel_ms(eng, stream, launch, iters, warmup):
    for _ in range(warmup):
        launch()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record(stream)
        launch()
        b.record(stream)
    eng.sync()
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    return {"median": round(float(np.median(ms)), 4), "min": round(float(ms.min()), 4), "max": round(float(ms.max()), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--wall-iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = device_info()
    stream = torch.cuda.Stream()
    eng = Engine(0, stream=stream.cuda_stream)
    res = {"device": dev, "shapes": {}, "wall_ms": {}, "kernel_ms": {}, "model_bytes": {}, "iters": a.iters,
           "warmup": a.warmup, "wall_iters": a.wall_iters}
    d_out = eng.dev_alloc(OUT_PIXELS * 12)
    for key, (w, h) in SHAPES.items():
        res["shapes"][key] = [w, h]
        rgb = np.random.RandomState(w + h).randint(0, 256, size=(h, w, 3)).astype(np.uint8)
        wall, kern, model = {}, {}, {}
        inputs = {fmt: layout(rgb, fmt) for fmt in FORMATS}
        f32 = eng.read_img_rgb8(rgb)                       # read_img's image: the f32 entry point's input
        want = {"rgb": eng.planet(f32)}
        coloured = int((want["rgb"][..., 0] >= 0).sum())
        for fmt, buf in list(inputs.items()) + [("f32", f32)]:
            if fmt == "f32":
                ref, call = want["rgb"], eng.planet
            else:
                ref = want["rgb"] if fmt != "grey" else eng.planet(eng.read_img_rgb8(buf))
                call = (lambda b, f=fmt: eng.planet_pix8(b, f))
            assert np.array_equal(call(buf).view(np.uint32), ref.view(np.uint32)), f"{key} {fmt}: planet differs"
            pin, ptr = pinned_copy(buf)
            try:
                assert np.array_equal(call(pin).view(np.uint32), ref.view(np.uint32))
                wall[fmt] = {"pageable": median_ms(lambda: call(buf), a.wall_iters, a.warmup),
                             "pinned": median_ms(lambda: call(pin), a.wall_iters, a.warmup)}
            finally:
                Engine.host_free(ptr)
            d_in = eng.dev_alloc(buf.nbytes)
            try:
                eng.dev_upload(d_in, buf)
                if fmt == "f32":
                    launch = (lambda: eng.planet_dev(d_in, w, h, d_out))
                else:
                    launch = (lambda f=fmt: eng.planet_pix8_dev(d_in, f, w, h, d_out))
                kern[f"{fmt}:{KERNEL[fmt]}"] = kernel_ms(eng, stream, launch, a.iters, a.warmup)
            finally:
                eng.dev_free(d_in)
            tap = 12 if fmt == "f32" else FORMATS[fmt]
            moved = OUT_PIXELS * (16 + 12) + coloured * 4 * tap
            model[fmt] = {"upload": buf.nbytes, "per_launch_upper_bound": moved,
                          "GBps_at_median": round(moved / (kern[f"{fmt}:{KERNEL[fmt]}"]["median"] * 1e-3) / 1e9, 1)}
        res["wall_ms"][key], res["kernel_ms"][key], res["model_bytes"][key] = wall, kern, model
        res["model_bytes"][key]["coloured_pixels"] = coloured
    eng.dev_free(d_out)
    eng.close()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
