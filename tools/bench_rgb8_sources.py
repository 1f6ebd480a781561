"""SIFT and the blend from 8-bit sources against the convert-then-f32 chain they replace, on the config 2 and config 5
shapes.  Old and new alternate in every repetition; medians are reported.

  python tools/bench_rgb8_sources.py [--configs 2,5] [--reps 5]

Rows per config:
  sift      convert (pano_rgb8_to_mat32f_batch_dev) + pano_sift_detect_batch_dev  vs  pano_sift_detect_batch_rgb8_dev
            (device 8-bit sources; device time up to the feature counts)
  blend     convert + pano_blend_dev  vs  pano_blend_rgb8_dev (device time)
  pipeline  one PipelinedStitcher(rgb8=True) job (pinned 8-bit in, cropped 8-bit mosaic out, wall time): the former
            chain (a per-slot f32 image block, the conversion launch, f32 SIFT and blend) vs the current one
`mark_gb` is the context pool's high-water mark (PANO_CACHE_MB=0): for sift / blend it includes the 8-bit device
sources, for pipeline the compute context's slot buffers.  Every new result is checked bit for bit against the old.
Prints one JSON line, with the card's name and power limit read in the same run.  Needs an H100."""
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

CONFIGS = {
    "2": dict(stack="ordered_13x1500x1112", bands=0, params=dict(ordered_input=1), max_output=None),
    "5": dict(stack="uav_64x4000x3000", bands=5, params=dict(ordered_input=1, multiband=5, lazy_read=0), max_output=8000),
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def run_config(key, reps, rows):
    import torch
    from openpano_b200 import synth
    from openpano_b200._abi import default_params
    from openpano_b200.capi import Engine
    from openpano_b200.stitcher import PipelinedStitcher, ordered_pairs, unpack_rgb8_mosaic

    cfg = CONFIGS[key]
    imgs, org = synth.config_stack(cfg["stack"])
    n, (h, w) = len(imgs), imgs[0].shape[:2]
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    del imgs
    items, geom = synth.translation_blend_setup(org, w, h, cfg["max_output"])
    params, bands = default_params(**cfg["params"]), cfg["bands"]
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    shapes, ws, hs, ch3 = [(h, w)] * n, [w] * n, [h] * n, [3] * n
    nb = h * w * 3
    out = {}

    def alternate(name, old, new, eng=None, check=None):
        """Warm both, then reps × (old, new), the order swapped every repetition: median times and the largest
        high-water marks."""
        res = {"old": ([], 0), "new": ([], 0)}
        for fn in (old, new):
            fn()
        for r in range(reps):
            for tag, fn in ((("old", old), ("new", new)) if r % 2 == 0 else (("new", new), ("old", old))):
                if eng is not None:
                    eng.sync()
                    eng.mem_high_water(reset=True)
                ms, mark = fn()
                if eng is not None:
                    mark = eng.mem_high_water()
                res[tag] = (res[tag][0] + [ms], max(res[tag][1], mark))
        if check is not None:
            check()
        row = dict(config=key, row=name)
        for tag in ("old", "new"):
            row[f"{tag}_ms"] = round(statistics.median(res[tag][0]), 3)
            row[f"{tag}_ms_all"] = [round(x, 2) for x in res[tag][0]]
            row[f"{tag}_mark_gb"] = round(res[tag][1] / 1e9, 3)
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)

    # ---- sift and blend on device sources
    stream = torch.cuda.Stream()
    eng = Engine(0, stream=stream.cuda_stream)
    d_pix = [eng.dev_alloc(nb) for _ in range(n)]
    for d, p in zip(d_pix, pix):
        eng.dev_upload(d, p)
    d_out = eng.dev_alloc(ow * oh * 12)

    def dev_timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        eng.sync()
        return e0.elapsed_time(e1), r

    feats = {}

    def sift_old():
        def body():
            d_f32 = [eng.dev_alloc(nb * 4) for _ in range(n)]
            eng.rgb8_to_mat32f_batch_dev(d_pix, ws, hs, ch3, d_f32)
            fs = eng.sift_detect_batch_ptr(d_f32, ws, hs, params, device=True)
            fs.count(0)
            for d in d_f32:
                eng.dev_free(d)
            return fs
        ms, fs = dev_timed(body)
        feats["old"] = fs.download(n - 1)
        fs.free()
        return ms, 0

    def sift_new():
        def body():
            fs = eng.sift_detect_batch_rgb8_ptr(d_pix, ws, hs, ch3, params, device=True)
            fs.count(0)
            return fs
        ms, fs = dev_timed(body)
        feats["new"] = fs.download(n - 1)
        fs.free()
        return ms, 0

    def sift_check():
        for a, b in zip(feats["old"], feats["new"]):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "sift from 8-bit differs"

    alternate("sift", sift_old, sift_new, eng, sift_check)
    mosaics = {t: np.empty((oh, ow, 3), np.float32) for t in ("old", "new")}

    def blend_old():
        def body():
            d_f32 = [eng.dev_alloc(nb * 4) for _ in range(n)]
            eng.rgb8_to_mat32f_batch_dev(d_pix, ws, hs, ch3, d_f32)
            eng.blend_dev(d_f32, shapes, items, geom, d_out, ow, oh, bands, params)
            for d in d_f32:
                eng.dev_free(d)
        ms, _ = dev_timed(body)
        eng.dev_download(mosaics["old"], d_out)
        return ms, 0

    def blend_new():
        ms, _ = dev_timed(lambda: eng.blend_rgb8_dev(d_pix, ch3, shapes, items, geom, d_out, ow, oh, bands, params))
        eng.dev_download(mosaics["new"], d_out)
        return ms, 0

    alternate("blend", blend_old, blend_new, eng,
              lambda: np.testing.assert_array_equal(mosaics["old"].view(np.uint32), mosaics["new"].view(np.uint32)))
    for d in d_pix + [d_out]:
        eng.dev_free(d)
    eng.close()

    # ---- one pipelined job: pinned 8-bit in, cropped 8-bit mosaic out
    pairs = ordered_pairs(n)
    host = [torch.from_numpy(p).pin_memory() for p in pix]
    hptr = [t.data_ptr() for t in host]
    new_ps = PipelinedStitcher(0, params, depth=2, rgb8=True, crop=True)
    old_ps = PipelinedStitcher(0, params, depth=2, rgb8=True, crop=True)
    outs = {t: torch.zeros(new_ps.out_bytes((ow, oh)), dtype=torch.uint8).pin_memory() for t in ("old", "new")}
    matches = {}
    f32_block = {}

    def old_run(ps, k):
        """PipelinedStitcher.run as it was before SIFT and the blend read 8-bit sources."""
        s = ps.slots[k]
        if k not in f32_block:
            f32_block[k] = ps.cmp.dev_alloc(n * nb * 4)
            ps.cmp.sync()
        ptrs = [f32_block[k] + q * nb * 4 for q in range(n)]
        ps.cmp.event_wait(s["ev_up"])
        ps.cmp.rgb8_to_mat32f_batch_dev([s["pix"] + o for o in s["pix_offs"]], ws, hs, ch3, ptrs)
        fs = ps.cmp.sift_detect_batch_ptr(ptrs, ws, hs, params, device=True)
        m = ps.cmp.match_pairs(fs, pairs, params)
        ps.cmp.event_wait(s["ev_dn"])
        ps.cmp.blend_dev(ptrs, shapes, items, geom, s["out"], ow, oh, bands, params)
        ps.cmp.crop_rect_dev(s["out"], ow, oh, s["out8"])
        ps.cmp.mat32f_to_rgb8_dev(s["out"], ow, oh, s["out8"], s["out8"] + ps.RGB8_HEADER)
        ps.cmp.event_record(s["ev_cmp"])
        fs.free()
        ps.dn.event_wait(s["ev_cmp"])
        ps.dn.dev_download_async(outs["old"].data_ptr(), s["out8"], ps.out_bytes((ow, oh)))
        ps.dn.event_record(s["ev_dn"])
        s["busy"] = True
        return (k, m)

    def job(tag):
        ps = old_ps if tag == "old" else new_ps
        ps.cmp.sync()
        ps.cmp.mem_high_water(reset=True)
        t0 = time.perf_counter()
        k = ps.stage(hptr, shapes, (ow, oh))
        handle = old_run(ps, k) if tag == "old" else ps.run(k, pairs, items, geom, outs["new"].data_ptr(), bands)
        matches[tag] = ps.wait(handle)
        ms = (time.perf_counter() - t0) * 1e3
        ps.cmp.sync()
        return ms, ps.cmp.mem_high_water()

    def pipe_check():
        # the header's rectangle and the cropped pixels; the rest of the buffer is not written
        old, new = (unpack_rgb8_mosaic(outs[t].numpy(), (ow, oh)) for t in ("old", "new"))
        assert old[0] == new[0] and np.array_equal(old[1], new[1]), "pipelined mosaic differs"
        assert all(np.array_equal(a, b) for a, b in zip(matches["old"], matches["new"])), "pipelined matches differ"

    alternate("pipeline", lambda: job("old"), lambda: job("new"), None, pipe_check)
    for k, d in f32_block.items():
        old_ps.cmp.dev_free(d)
    old_ps.close()
    new_ps.close()
    out.update(n=n, w=w, h=h, canvas=[ow, oh], bands=bands, u8_source_gb=round(n * nb / 1e9, 3),
               f32_copy_gb=round(4 * n * nb / 1e9, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="2,5")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    os.environ["PANO_CACHE_MB"] = "0"
    info = gpu_info()
    rows, shapes = [], {}
    for key in a.configs.split(","):
        shapes[key] = run_config(key, a.reps, rows)
    print(json.dumps(dict(**info, reps=a.reps, configs=shapes, rows=rows)))


if __name__ == "__main__":
    main()
