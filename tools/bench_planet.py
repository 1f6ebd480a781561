#!/usr/bin/env python
"""Cost of the little-planet view, planet() (main.cc:294-331), on the engine.  One JSON line:

  device            card name and power limit, read by one nvidia-smi call in this run
  first_call_ms     host wall time of the first pano_planet_dev of the process (host table build + upload + kernel,
                    then a stream sync), and of the first call on a second context (upload + kernel only)
  planet_dev_ms     per input shape: device time of pano_planet_dev between CUDA events on the engine's stream,
                    median (and min / max) of --iters calls after --warmup calls
  planet_wall_ms    per input shape: host wall time of pano_planet (upload of the f32 mosaic, kernel, download of the
                    12 MB result), median of --wall-iters calls
  model_bytes       per input shape: 16 B of table + 12 B of output per output pixel, plus 4 taps x 12 B per coloured
                    pixel (an upper bound on the gathers: neighbouring pixels share taps), and the rate they imply
  ref_cpu_ms        per input shape: the reference's own planet() (oracle/_ref/libopenpano_ref_planet.so, one
                    thread, -O2), median of --ref-iters calls; null when that checker was not built

    python tools/bench_planet.py [--iters 200] [--warmup 20] [--out results/bench_planet.jsonl]
"""
from __future__ import annotations

import argparse
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
from tests import planet_util as pu  # noqa: E402

SHAPES = [(8000, 1449, "mosaic"), (1800, 300, "band")]     # the CMU1 mosaic (run_test.py) and a small pano
OUT_PIXELS = pu.SIZE * pu.SIZE


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": "not available", "error": str(e)}


def first_calls(img):
    """Wall time of the first planet of the process and of the first one on another context."""
    h, w = img.shape[:2]
    out = {}
    for tag in ("process", "second_context"):
        eng = Engine(0)
        d_src, d_out = eng.dev_alloc(img.nbytes), eng.dev_alloc(OUT_PIXELS * 12)
        eng.dev_upload(d_src, img)
        eng.sync()
        t0 = time.perf_counter()
        eng.planet_dev(d_src, w, h, d_out)
        eng.sync()
        out[tag] = round((time.perf_counter() - t0) * 1e3, 3)
        eng.dev_free(d_src)
        eng.dev_free(d_out)
        eng.close()
    return out


def device_times(eng, stream, img, iters, warmup):
    h, w = img.shape[:2]
    d_src, d_out = eng.dev_alloc(img.nbytes), eng.dev_alloc(OUT_PIXELS * 12)
    try:
        eng.dev_upload(d_src, img)
        for _ in range(warmup):
            eng.planet_dev(d_src, w, h, d_out)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
        for a, b in ev:
            a.record(stream)
            eng.planet_dev(d_src, w, h, d_out)
            b.record(stream)
        eng.sync()
        ms = np.array([a.elapsed_time(b) for a, b in ev])
    finally:
        eng.dev_free(d_src)
        eng.dev_free(d_out)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--wall-iters", type=int, default=20)
    ap.add_argument("--ref-iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = device_info()
    imgs = {(w, h): pu.make_input(w, h, 1, holes) for w, h, holes in SHAPES}
    first = first_calls(imgs[SHAPES[0][:2]])

    stream = torch.cuda.Stream()
    eng = Engine(0, stream=stream.cuda_stream)
    res = {"device": dev, "first_call_ms": first, "planet_dev_ms": {}, "planet_wall_ms": {}, "model_bytes": {},
           "ref_cpu_ms": {}, "iters": a.iters, "warmup": a.warmup}
    for (w, h), img in imgs.items():
        key = f"{w}x{h}"
        ms = device_times(eng, stream, img, a.iters, a.warmup)
        med = float(np.median(ms))
        res["planet_dev_ms"][key] = {"median": round(med, 4), "min": round(float(ms.min()), 4),
                                     "max": round(float(ms.max()), 4)}
        for _ in range(3):
            out = eng.planet(img)
        wall = []
        for _ in range(a.wall_iters):
            t0 = time.perf_counter()
            eng.planet(img)
            wall.append(time.perf_counter() - t0)
        res["planet_wall_ms"][key] = round(float(np.median(wall)) * 1e3, 3)
        coloured = int((out[..., 0] >= 0).sum())
        nbytes = OUT_PIXELS * (16 + 12) + coloured * 4 * 12
        res["model_bytes"][key] = {"table_and_output": OUT_PIXELS * 28, "gathers_upper_bound": coloured * 48,
                                   "coloured_pixels": coloured, "input_bytes": img.nbytes,
                                   "GBps_at_median": round(nbytes / (med * 1e-3) / 1e9, 1)}
        if pu.have_ref():
            t = []
            for _ in range(a.ref_iters):
                t0 = time.perf_counter()
                pu.ref_planet(img)
                t.append(time.perf_counter() - t0)
            res["ref_cpu_ms"][key] = round(float(np.median(t)) * 1e3, 2)
        else:
            res["ref_cpu_ms"][key] = None
    eng.close()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
