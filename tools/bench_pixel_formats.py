"""What the decoders' layouts cost: SIFT from lodepng's RGBA (PANO_PIX_RGBA) and CImg's planes (PANO_PIX_RGB_PLANAR)
against interleaved RGB, end to end through the SIFT stream and per kernel.

  python tools/bench_pixel_formats.py                          # both parts
  python tools/bench_pixel_formats.py --part stream --n 16     # fewer config 5 views

Part `stream`: config 5 (64 × 4000×3000) from pinned host buffers through pano_sift_stream, windows of 1, until the
featureset's counts are on the host.  Rows:
  rgb direct         interleaved RGB sources (3 B/px), today's path
  rgba direct        the decoder's RGBA buffers sent as they are (4 B/px)
  rgba strip+rgb     the RGBA buffers stripped to RGB on the host first (numpy, one image ahead of its add, into
                     pinned buffers), the host pass inside the timed window
  planar direct      CImg's planes sent as they are (3 B/px)
  strip only         the host pass alone over all images
Wall ms, median over --reps after one warm-up; every featureset is checked bit for bit against rgb direct's.
Part `kernels`: device-resident grey, RGB, RGBA and planar sources of configs 2 and 5 (--views5 of config 5's
views), per-launch times (eng profiling: CUDA events around each launch, median-free mean over --reps calls) of
every kernel that reads 8-bit sources: k_pyramid_grey (SIFT batch), k_linear_blend (blend_rgb8_dev, bands 0),
k_linear_accumulate (a blend stream of device sources, windows of 1), k_mb_first_level (MULTIBAND 2),
k_cyl_warp_batch and k_planet8 (each source image as the mosaic).  Each row names the profile entry it read: the
one kernel the call launched whose name starts with the kernel's, so the same script times builds that name their
8-bit instantiations differently (PANO_B200_LIB picks the build).  Prints one JSON line per row and a summary line
with the card's name and power limit read in the same run.  Needs an H100."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import numpy as np  # noqa: E402

CONFIGS = {"2": "ordered_13x1500x1112", "5": "uav_64x4000x3000"}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def emit(row):
    print(json.dumps(row), flush=True)
    return row


def stream_part(a, rows):
    import torch
    from openpano_b200 import synth
    from openpano_b200.capi import PIX_RGB, PIX_RGB_PLANAR, PIX_RGBA, SRC_RGB8_HOST, Engine

    imgs, _ = synth.config_stack(CONFIGS["5"], a.n)
    n, (h, w) = len(imgs), imgs[0].shape[:2]
    rgb = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    del imgs
    rgba = [torch.empty((h, w, 4), dtype=torch.uint8).pin_memory() for _ in range(n)]
    for t, x in zip(rgba, rgb):
        v = t.numpy()
        v[..., :3] = x
        v[..., 3] = 255
    pinned = [torch.empty((h, w, 3), dtype=torch.uint8).pin_memory() for _ in range(n)]   # RGB, then planes
    eng = Engine(0)

    def run(ptrs, fmt, before_add=None):
        s = eng.sift_stream([(h, w)] * n)
        try:
            for k in range(n):
                if before_add:
                    before_add(k)
                s.add([ptrs[k]], SRC_RGB8_HOST, fmt)
            fs = s.finish()
        finally:
            s.close()
        fs.count(0)
        return fs

    def timed(fn):
        fn().free()
        wall, fs = [], None
        for _ in range(a.reps):
            if fs is not None:
                fs.free()
            eng.sync()
            t0 = time.perf_counter()
            fs = fn()
            eng.sync()
            wall.append((time.perf_counter() - t0) * 1e3)
        return statistics.median(wall), fs

    def same(fs, want):
        return all(fs.download(i)[0].tobytes() == want.download(i)[0].tobytes() and
                   fs.download(i)[1].tobytes() == want.download(i)[1].tobytes() for i in range(n))

    def strip(k):
        np.copyto(pinned[k].numpy(), rgba[k].numpy()[..., :3])

    for t, x in zip(pinned, rgb):
        t.numpy()[...] = x
    t_rgb, want = timed(lambda: run([t.data_ptr() for t in pinned], PIX_RGB))
    rows.append(emit(dict(part="stream", row="rgb direct", wall_ms=round(t_rgb, 1), h2d_gb=round(n * h * w * 3 / 1e9, 3))))
    t, fs = timed(lambda: run([t.data_ptr() for t in rgba], PIX_RGBA))
    rows.append(emit(dict(part="stream", row="rgba direct", wall_ms=round(t, 1), h2d_gb=round(n * h * w * 4 / 1e9, 3),
                          same=same(fs, want))))
    fs.free()
    t, fs = timed(lambda: run([t.data_ptr() for t in pinned], PIX_RGB, before_add=strip))
    rows.append(emit(dict(part="stream", row="rgba strip+rgb", wall_ms=round(t, 1),
                          h2d_gb=round(n * h * w * 3 / 1e9, 3), same=same(fs, want))))
    fs.free()
    strip_ms = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        for k in range(n):
            strip(k)
        strip_ms.append((time.perf_counter() - t0) * 1e3)
    rows.append(emit(dict(part="stream", row="strip only", wall_ms=round(statistics.median(strip_ms), 1))))
    for t_, x in zip(pinned, rgb):
        t_.numpy().reshape(3, h, w)[...] = np.moveaxis(x, 2, 0)
    t, fs = timed(lambda: run([t.data_ptr() for t in pinned], PIX_RGB_PLANAR))
    rows.append(emit(dict(part="stream", row="planar direct", wall_ms=round(t, 1), h2d_gb=round(n * h * w * 3 / 1e9, 3),
                          same=same(fs, want))))
    fs.free()
    want.free()
    eng.close()
    return dict(n=n, w=w, h=h)


def kernel_part(a, rows):
    from openpano_b200 import synth
    from openpano_b200._abi import default_params
    from openpano_b200.capi import PIX_FORMATS, SRC_RGB8_DEV, Engine

    eng = Engine(0)
    for cfg in ("2", "5"):
        imgs, org = synth.config_stack(CONFIGS[cfg], a.views5 if cfg == "5" else None)
        n, (h, w) = len(imgs), imgs[0].shape[:2]
        rgb = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
        del imgs
        bufs = {"grey": [np.ascontiguousarray(x[..., 0]) for x in rgb], "rgb": rgb,
                "rgba": [np.concatenate([x, np.full((h, w, 1), 255, np.uint8)], 2) for x in rgb],
                "planar": [np.ascontiguousarray(np.moveaxis(x, 2, 0)) for x in rgb]}
        items, geom = synth.translation_blend_setup(org, w, h)
        tw, th = max(it[2] for it in items), max(it[3] for it in items)
        p = default_params()
        pb = default_params(multiband=2)
        ow, oh = eng.cyl_warp_shape(w, h, 1.0, p)[:2]
        d_out = eng.dev_alloc(max(tw * th, ow * oh * n, Engine.PLANET_SIZE ** 2) * 12)
        warp_out = [d_out + k * ow * oh * 12 for k in range(n)]

        def stream_blend(d_src, code):
            s = eng.blend_stream([(h, w)] * n, items, geom, 0, p)
            try:
                for d in d_src:
                    s.add([d], SRC_RGB8_DEV, code)
                s.finish_dev(d_out)
            finally:
                s.close()

        for fmt, code in PIX_FORMATS.items():
            d_src = [eng.dev_alloc(x.nbytes) for x in bufs[fmt]]
            for d, x in zip(d_src, bufs[fmt]):
                eng.dev_upload(d, x)
            ch = [code] * n
            # kernel -> a call that launches it; the profile entry is the one name that starts with the kernel's
            ops = {
                "k_pyramid_grey": lambda: eng.sift_detect_batch_rgb8_ptr(d_src, [w] * n, [h] * n, ch, p, device=True).free(),
                "k_linear_blend": lambda: eng.blend_rgb8_dev(d_src, ch, [(h, w)] * n, items, geom, d_out, tw, th, 0, p),
                "k_linear_accumulate": lambda: stream_blend(d_src, code),
                "k_mb_first_level": lambda: eng.blend_rgb8_dev(d_src, ch, [(h, w)] * n, items, geom, d_out, tw, th, 2, pb),
                "k_cyl_warp": lambda: eng.cyl_warp_batch_rgb8_dev(d_src, ch, [(h, w)] * n, warp_out, None, 1.0, p),
                "k_planet": lambda: [eng.planet_pix8_dev(d, code, w, h, d_out) for d in d_src],
            }
            for kernel, op in ops.items():
                op()
                eng.sync()
                eng.profile(True)
                eng.profile_reset()
                for _ in range(a.reps):
                    op()
                eng.sync()
                prof = eng.profile_read()
                eng.profile(False)
                name = [k for k in prof if k.startswith(kernel)]
                assert len(name) == 1, (kernel, fmt, sorted(prof))
                launches, ms = prof[name[0]]
                rows.append(emit(dict(part="kernels", config=cfg, n=n, w=w, h=h, kernel=name[0], source=fmt,
                                      ms_per_launch=round(ms / launches, 3), launches=launches)))
            for d in d_src:
                eng.dev_free(d)
        eng.dev_free(d_out)
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=["stream", "kernels", "all"], default="all")
    ap.add_argument("--n", type=int, default=64, help="config 5 views of the stream part")
    ap.add_argument("--views5", type=int, default=8, help="config 5 views of the kernel part")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    rows, shape = [], None
    if a.part in ("stream", "all"):
        shape = stream_part(a, rows)
    if a.part in ("kernels", "all"):
        kernel_part(a, rows)
    print(json.dumps(dict(**gpu_info(), stream_shape=shape, rows=rows)))


if __name__ == "__main__":
    main()
