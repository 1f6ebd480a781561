"""The cylinder warp and the row strips of the composite from 8-bit sources against the convert-then-f32 work they
replace.  Old and new alternate in one process; medians are reported.

  python tools/bench_rgb8_warp_strips.py [--chain 1,2] [--chain-reps 20] [--strips 8] [--strip-reps 10]

Rows:
  chain   cylinder mode's device chain on one GPU: SIFT -> adjacent-pair matches -> warp of every image and its
          keypoints -> LinearBlender composite of the warped images.  old: convert every image to f32
          (pano_rgb8_to_mat32f_batch_dev) and run the f32 chain; new: SIFT and the warp read the 8-bit pixels
          (pano_sift_detect_batch_rgb8_dev, pano_cyl_warp_batch_rgb8_dev).  At config 1's shape (8 × 600×400) and
          at 13 × 1500×1112 (config 2's views).  The chain's time includes its host round trips (match lists,
          keypoints); its `warp` entry times the warp alone, ten launches per window: convert + f32 warp vs the
          8-bit warp.
  strip   config 5's 64 × 4000×3000 5-band composite as row strips, one after another on one GPU.  old: what
          DistributedStitcher.run_rgb8 did per strip — convert the images whose ROI lies within 256 rows of the
          strip, then pano_blend_rows_dev; new: pano_blend_rows_rgb8_dev on the 8-bit sources.
`mark_gb` is the context pool's high-water mark (PANO_CACHE_MB=0), 8-bit device sources included.  Every new result
is checked bit for bit against the old.  Prints one JSON line, with the card's name and power limit read in the same
run.  Needs an H100."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import numpy as np  # noqa: E402

CHAINS = {"1": "cmu0_8x600x400", "2": "ordered_13x1500x1112"}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


class Bench:
    def __init__(self):
        import torch
        from openpano_b200.capi import Engine
        self.torch = torch
        self.stream = torch.cuda.Stream()
        self.eng = Engine(0, stream=self.stream.cuda_stream)

    def timed(self, fn):
        """Device time of fn's work on the engine's stream and the pool's high-water mark during it."""
        torch, eng = self.torch, self.eng
        eng.sync()
        eng.mem_high_water(reset=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(self.stream)
        r = fn()
        e1.record(self.stream)
        eng.sync()
        return e0.elapsed_time(e1), eng.mem_high_water(), r


def alternate(reps, old, new):
    """Warm both, then reps × (old, new), the order swapped every repetition: {tag: (times, largest mark)}."""
    res = {"old": ([], 0), "new": ([], 0)}
    old()
    new()
    for r in range(reps):
        for tag, fn in ((("old", old), ("new", new)) if r % 2 == 0 else (("new", new), ("old", old))):
            ms, mark = fn()
            res[tag] = (res[tag][0] + [ms], max(res[tag][1], mark))
    return res


def summarise(row, res):
    for tag in ("old", "new"):
        row[f"{tag}_ms"] = round(statistics.median(res[tag][0]), 3)
        row[f"{tag}_ms_all"] = [round(x, 2) for x in res[tag][0]]
        row[f"{tag}_mark_gb"] = round(res[tag][1] / 1e9, 3)
    print(json.dumps(row), file=sys.stderr, flush=True)
    return row


def run_chain(b, key, reps):
    from openpano_b200 import synth
    from openpano_b200._abi import default_params

    eng = b.eng
    views, org = synth.config_stack(CHAINS[key])
    n, (h, w) = len(views), views[0].shape[:2]
    pix = [(v * 255.0 + 0.5).astype(np.uint8) for v in views]
    del views
    p = default_params(ordered_input=1)
    pairs = [(k, k + 1) for k in range(n - 1)]
    ws, hs, ch3, nb = [w] * n, [h] * n, [3] * n, h * w * 3
    ow, oh, _, _ = eng.cyl_warp_shape(w, h, 1.0, p)
    items, geom = synth.translation_blend_setup(org, ow, oh)
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    d_pix = [eng.dev_alloc(nb) for _ in range(n)]
    for d, x in zip(d_pix, pix):
        eng.dev_upload(d, x)
    d_warp = [eng.dev_alloc(ow * oh * 12) for _ in range(n)]
    d_out = eng.dev_alloc(tw * th * 12)
    got = {}

    def chain(rgb8):
        d_f32 = None
        if rgb8:
            fs = eng.sift_detect_batch_rgb8_ptr(d_pix, ws, hs, ch3, p, device=True)
        else:
            d_f32 = [eng.dev_alloc(nb * 4) for _ in range(n)]
            eng.rgb8_to_mat32f_batch_dev(d_pix, ws, hs, ch3, d_f32)
            fs = eng.sift_detect_batch_ptr(d_f32, ws, hs, p, device=True)
        m = eng.match_pairs(fs, pairs, p)
        kp = [np.ascontiguousarray(fs.download(i)[0]).copy() for i in range(n)]
        fs.free()
        if rgb8:
            eng.cyl_warp_batch_rgb8_dev(d_pix, ch3, [(h, w)] * n, d_warp, kp, 1.0, p)
        else:
            eng.cyl_warp_batch_dev(d_f32, [(h, w)] * n, d_warp, kp, 1.0, p)
            for d in d_f32:
                eng.dev_free(d)
        eng.blend_dev(d_warp, [(oh, ow)] * n, items, geom, d_out, tw, th, 0, p)
        return m, kp

    def step(tag):
        ms, mark, (m, kp) = b.timed(lambda: chain(tag == "new"))
        mosaic = np.empty((th, tw, 3), np.float32)
        warped0 = np.empty((oh, ow, 3), np.float32)
        eng.dev_download(mosaic, d_out)
        eng.dev_download(warped0, d_warp[0])
        got[tag] = (m, kp, mosaic, warped0)
        return ms, mark

    res = alternate(reps, lambda: step("old"), lambda: step("new"))

    def warp_only(tag, launches=10):
        """The warp alone, `launches` times in one window: convert + f32 warp vs the 8-bit warp."""
        def body():
            for _ in range(launches):
                if tag == "old":
                    d_f32 = [eng.dev_alloc(nb * 4) for _ in range(n)]
                    eng.rgb8_to_mat32f_batch_dev(d_pix, ws, hs, ch3, d_f32)
                    eng.cyl_warp_batch_dev(d_f32, [(h, w)] * n, d_warp, None, 1.0, p)
                    for d in d_f32:
                        eng.dev_free(d)
                else:
                    eng.cyl_warp_batch_rgb8_dev(d_pix, ch3, [(h, w)] * n, d_warp, None, 1.0, p)
        ms, mark, _ = b.timed(body)
        return ms / launches, mark

    res_w = alternate(reps, lambda: warp_only("old"), lambda: warp_only("new"))
    warp_row = summarise(dict(row="warp", stack=CHAINS[key]), res_w)
    (mo, ko, so, wo), (mn, kn, sn, wn) = got["old"], got["new"]
    assert len(mo) == len(mn) and all(np.array_equal(a, c) for a, c in zip(mo, mn)), "matches differ"
    assert all(a.tobytes() == c.tobytes() for a, c in zip(ko, kn)), "warped keypoints differ"
    assert wo.tobytes() == wn.tobytes() and so.tobytes() == sn.tobytes(), "warped image or mosaic differs"
    for d in d_pix + d_warp + [d_out]:
        eng.dev_free(d)
    row = dict(row="chain", stack=CHAINS[key], n=n, w=w, h=h, warp=[ow, oh], canvas=[tw, th],
               f32_copy_gb=round(4 * n * nb / 1e9, 3), identical=True)
    row = summarise(row, res)
    row["warp"] = warp_row
    return row


def run_strips(b, n_strips, reps):
    from openpano_b200 import synth
    from openpano_b200._abi import default_params

    eng = b.eng
    views, org = synth.config_stack("uav_64x4000x3000")
    n, (h, w) = len(views), views[0].shape[:2]
    pix = [(v * 255.0 + 0.5).astype(np.uint8) for v in views]
    del views
    items, geom = synth.translation_blend_setup(org, w, h, 8000)
    bands, p = 5, default_params(ordered_input=1, multiband=5, lazy_read=0)
    shapes, ch3, nb = [(h, w)] * n, [3] * n, h * w * 3
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    rows_per = (th + n_strips - 1) // n_strips
    cuts = [(min(th, s * rows_per), min(th, (s + 1) * rows_per)) for s in range(n_strips)]
    d_pix = [eng.dev_alloc(nb) for _ in range(n)]
    for d, x in zip(d_pix, pix):
        eng.dev_upload(d, x)
    del pix
    d_strip = eng.dev_alloc(rows_per * tw * 12)
    out = {t: np.empty((th, tw, 3), np.float32) for t in ("old", "new")}
    n_conv = []

    def strip_old(r0, r1):
        need = [k for k in range(n) if items[k][1] <= r1 + 256 and items[k][3] >= r0 - 256]
        block = eng.dev_alloc(max(len(need), 1) * nb * 4)
        ptrs = [block] * n                     # images that cannot reach the strip: any valid pointer
        if need:
            dst = [block + q * nb * 4 for q in range(len(need))]
            eng.rgb8_to_mat32f_batch_dev([d_pix[k] for k in need], [w] * len(need), [h] * len(need),
                                         [3] * len(need), dst)
            for q, k in enumerate(need):
                ptrs[k] = dst[q]
        eng.blend_rows_dev(ptrs, shapes, items, geom, d_strip, tw, th, r0, r1, bands, p)
        eng.dev_free(block)
        return len(need)

    def strip_new(r0, r1):
        eng.blend_rows_rgb8_dev(d_pix, ch3, shapes, items, geom, d_strip, tw, th, r0, r1, bands, p)

    per = []
    for s, (r0, r1) in enumerate(cuts):
        def one(tag):
            ms, mark, k = b.timed(lambda: strip_old(r0, r1) if tag == "old" else strip_new(r0, r1))
            eng.dev_download(out[tag][r0:r1], d_strip)
            if tag == "old":
                n_conv.append(k)
            return ms, mark
        res = alternate(reps, lambda: one("old"), lambda: one("new"))
        per.append(summarise(dict(row="strip", strip=s, rows=[r0, r1], converted_images=n_conv[-1]), res))
    assert out["old"].tobytes() == out["new"].tobytes(), "strips differ"
    for d in d_pix + [d_strip]:
        eng.dev_free(d)
    return dict(row="strips", n=n, w=w, h=h, canvas=[tw, th], bands=bands, strips=n_strips, identical=True,
                old_ms_total=round(sum(r["old_ms"] for r in per), 3), new_ms_total=round(sum(r["new_ms"] for r in per), 3),
                old_mark_gb_max=max(r["old_mark_gb"] for r in per), new_mark_gb_max=max(r["new_mark_gb"] for r in per),
                u8_source_gb=round(n * nb / 1e9, 3), per_strip=per)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chain", default="1,2")
    ap.add_argument("--chain-reps", type=int, default=20)
    ap.add_argument("--strips", type=int, default=8)
    ap.add_argument("--strip-reps", type=int, default=10)
    a = ap.parse_args()
    os.environ["PANO_CACHE_MB"] = "0"
    info = gpu_info()
    b = Bench()
    rows = [run_chain(b, key, a.chain_reps) for key in a.chain.split(",") if key]
    if a.strips > 0:
        rows.append(run_strips(b, a.strips, a.strip_reps))
    b.eng.close()
    print(json.dumps(dict(**info, chain_reps=a.chain_reps, strip_reps=a.strip_reps, rows=rows)))


if __name__ == "__main__":
    main()
