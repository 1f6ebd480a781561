"""SIFT of a device-resident batch with two builds of the library, alternated: the batch time and the per-kernel
times of the pyramid's front end (the grey plane of every octave), on the config 2, 3 and 5 shapes, from f32 and
from 8-bit sources.

  python tools/bench_pyramid_grey.py --old openpano_b200/_variants/parent.so [--new LIB] [--configs 2,3,5]
                                     [--reps 11] [--config5-views 16]

Each build runs in a worker process of its own (PANO_B200_LIB names the library), so both hold their buffers
at once and take turns on the GPU: every repetition times one batch on each, the order swapped every repetition.
Rows per (config, source):
  batch_ms   CUDA events around one pano_sift_detect_batch[_rgb8]_dev call (every launch of the batch and the
             count copy), median of --reps
  kernels    eng.profile times of the kernels that build the grey planes (k_working_resize[_rgb8] +
             k_octave_grey, or k_pyramid_grey[_rgb8]), median of --reps profiled batches
  same       both builds give the same bytes for every image's coordinates and descriptors
8-bit sources are the generator's pixels as read_img would receive them; the f32 sources are their read_img
conversion (pano_rgb8_to_mat32f_batch_dev).  Config 5 uses the first --config5-views of its 64 views: generating
all of them takes minutes of host time, and the per-image work is the same.  Prints one JSON line, with the
card's name and power limit read in the same run.  Needs an H100."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402

CONFIGS = {"2": "ordered_13x1500x1112", "3": "unordered_38x1300x867", "5": "uav_64x4000x3000"}
FRONT = ("k_working_resize", "k_working_resize_rgb8", "k_octave_grey", "k_pyramid_grey", "k_pyramid_grey_rgb8")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


# ----------------------------------------------------------------------------- worker (one build of the library)
def worker():
    out = os.fdopen(os.dup(1), "w")     # replies only; anything else the process prints goes to stderr
    os.dup2(2, 1)
    import torch
    from openpano_b200._abi import default_params
    from openpano_b200.capi import Engine

    stream = torch.cuda.Stream()
    eng = Engine(0, stream=stream.cuda_stream)
    params = default_params()
    st = {}

    def sift(src):
        if src == "f32":
            return eng.sift_detect_batch_ptr(st["f32"], st["ws"], st["hs"], params, device=True)
        return eng.sift_detect_batch_rgb8_ptr(st["u8"], st["ws"], st["hs"], [3] * st["n"], params, device=True)

    def timed(src):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fs = sift(src)
        e1.record(stream)
        fs.count(0)
        e1.synchronize()
        fs.free()
        return e0.elapsed_time(e1)

    for line in sys.stdin:
        cmd = json.loads(line)
        op = cmd["cmd"]
        if op == "load":
            n, w, h = cmd["n"], cmd["w"], cmd["h"]
            pix = np.load(cmd["path"], mmap_mode="r")
            st.update(n=n, ws=[w] * n, hs=[h] * n, u8=[eng.dev_alloc(h * w * 3) for _ in range(n)],
                      f32=[eng.dev_alloc(h * w * 12) for _ in range(n)])
            for d, k in zip(st["u8"], range(n)):
                eng.dev_upload(d, np.ascontiguousarray(pix[k]))
            eng.rgb8_to_mat32f_batch_dev(st["u8"], st["ws"], st["hs"], [3] * n, st["f32"])
            for src in ("f32", "u8", "f32", "u8"):          # warm-up: pool, function attributes, list capacity
                timed(src)
            reply = {"ok": True}
        elif op == "time":
            reply = {"ms": timed(cmd["src"])}
        elif op == "profile":
            eng.profile(True)
            eng.profile_reset()
            fs = sift(cmd["src"])
            fs.count(0)
            prof = eng.profile_read()
            eng.profile(False)
            fs.free()
            reply = {"kernels": {k: v[1] for k, v in prof.items()}}
        elif op == "digest":
            fs = sift(cmd["src"])
            hsh = hashlib.sha256()
            for i in range(st["n"]):
                c, d = fs.download(i)
                hsh.update(c.tobytes())
                hsh.update(d.tobytes())
            fs.free()
            reply = {"sha256": hsh.hexdigest()}
        elif op == "free":
            for d in st["u8"] + st["f32"]:
                eng.dev_free(d)
            eng.sync()
            st.clear()
            reply = {"ok": True}
        else:
            break
        print(json.dumps(reply), file=out, flush=True)
    eng.close()


class Worker:
    def __init__(self, lib):
        env = dict(os.environ)
        if lib:
            env["PANO_B200_LIB"] = str(Path(lib).resolve())
        else:
            env.pop("PANO_B200_LIB", None)
        self.p = subprocess.Popen([sys.executable, __file__, "--worker"], stdin=subprocess.PIPE, stdout=subprocess.PIPE,
                                  text=True, env=env)

    def send(self, **cmd):
        self.p.stdin.write(json.dumps(cmd) + "\n")
        self.p.stdin.flush()

    def recv(self):
        line = self.p.stdout.readline()
        if not line:
            raise SystemExit(f"worker exited with {self.p.wait()}")
        return json.loads(line)

    def call(self, **cmd):
        self.send(**cmd)
        return self.recv()

    def close(self):
        self.send(cmd="quit")
        self.p.stdin.close()
        self.p.wait()


def front_ms(kernels):
    return sum(v for k, v in kernels.items() if k in FRONT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old", help="library of the parent build (required)")
    ap.add_argument("--new", default=None, help="library of this build (default: the in-tree build)")
    ap.add_argument("--configs", default="2,3,5")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--config5-views", type=int, default=16)
    ap.add_argument("--worker", action="store_true")
    a = ap.parse_args()
    if a.worker:
        worker()
        return
    if not a.old:
        ap.error("--old is required")
    from tools.bench_configs import quantise
    from openpano_b200 import synth

    info = gpu_info()
    builds = {"old": Worker(a.old), "new": Worker(a.new)}
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for key in a.configs.split(","):
            views, _ = synth.config_stack(CONFIGS[key], n=a.config5_views if key == "5" else None)
            pix = np.stack(quantise(views))
            del views
            n, h, w = pix.shape[:3]
            path = os.path.join(tmp, f"pix{key}.npy")
            np.save(path, pix)
            del pix
            for wk in builds.values():
                wk.send(cmd="load", path=path, n=n, w=w, h=h)
            for wk in builds.values():
                assert wk.recv()["ok"]
            os.unlink(path)
            for src in ("f32", "u8"):
                ms = {"old": [], "new": []}
                kern = {"old": [], "new": []}
                for r in range(a.reps):
                    order = ("old", "new") if r % 2 == 0 else ("new", "old")
                    for tag in order:
                        ms[tag].append(builds[tag].call(cmd="time", src=src)["ms"])
                    for tag in order:
                        kern[tag].append(builds[tag].call(cmd="profile", src=src)["kernels"])
                same = builds["old"].call(cmd="digest", src=src)["sha256"] == builds["new"].call(cmd="digest", src=src)["sha256"]
                row = dict(config=key, images=n, image_wh=[w, h], src=src, same=same)
                for tag in ("old", "new"):
                    names = sorted({k for kd in kern[tag] for k in kd if k in FRONT})
                    row[f"{tag}_batch_ms"] = round(statistics.median(ms[tag]), 4)
                    row[f"{tag}_batch_ms_all"] = [round(x, 3) for x in ms[tag]]
                    row[f"{tag}_front_ms"] = round(statistics.median(front_ms(kd) for kd in kern[tag]), 4)
                    row[f"{tag}_front_kernels_ms"] = {k: round(statistics.median(kd.get(k, 0.0) for kd in kern[tag]), 4)
                                                      for k in names}
                rows.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
            for wk in builds.values():
                assert wk.call(cmd="free")["ok"]
    for wk in builds.values():
        wk.close()
    print(json.dumps(dict(**info, reps=a.reps, old=a.old, new=a.new or "in-tree", rows=rows)))


if __name__ == "__main__":
    main()
