"""Per-config measurement legs of bench.py (BASELINE.json configs 1-5) and the sharded
multi-GPU leg (SURVEY.md §8e).  bench.py imports this; nothing here is on the product path.

Every stack leg reports, for one pass of the hot path over the named stack:
  ms_device      device-resident step (inputs already f32 in HBM), CUDA events, median of K
  e2e_ms         one job through host buffers: pinned 8-bit pixels in -> u8->f32, SIFT, match
                 lists back to the host, blend, crop + 8-bit mosaic out (H2D / D2H inside)
  kernels        event-timed per-kernel times of one step with the §8d algorithmic bytes
  roofline       the dominant kernel of that step against the measured peaks
  parity_sample  a bounded check against the oracle port (image 0's features, pair 0's matches)
  cpu_baseline   the reference's own TUs (oracle/_ref, OpenMP, all host cores) on a bounded sample
"""
from __future__ import annotations

import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


# ----------------------------------------------------------------------------- byte model
def octave_dims(w, h, params):
    """Working/octave sizes with the reference's float arithmetic (feature.cc:33-34, dog.cc:105-107)."""
    f32 = np.float32
    ratio = f32(params.sift_working_size) * f32(2.0) / f32(w + h)
    h0, w0 = int(f32(h) * ratio), int(f32(w) * ratio)
    dims = [(w0, h0)]
    for o in range(1, params.num_octave):
        factor = f32(float(params.scale_factor) ** (-o))
        dims.append((int(np.ceil(f32(w0) * factor)), int(np.ceil(f32(h0) * factor))))
    return dims


def algorithmic_bytes(shapes, items, params, counts, bands):
    """Per-launch algorithmic traffic of each kernel (compulsory-traffic model of
    SURVEY.md §8d: every array one stage produces and another consumes is written
    once and read once; fused temporaries are free).  shapes: (h, w) per image."""
    ns = params.num_scale
    p_in = sum(h * w for h, w in shapes)
    p0 = sp = 0
    for (h, w) in shapes:
        d = octave_dims(w, h, params)
        p0 += d[0][0] * d[0][1]
        sp += sum(a * b for a, b in d)
    n_desc = sum(counts)
    roi = sum((it[2] - it[0] + 1) * (it[3] - it[1] + 1) for it in items)
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    return {
        "k_rgb8_to_f32": p_in * 15,
        # the source's bilinear taps (at most 4 per working pixel) in, every octave's grey plane out; the
        # working RGB image is a shared-memory tile.  8-bit sources: 3 B per tap pixel (1 for grey ones)
        "k_pyramid_grey": min(p_in, 4 * p0) * 12 + sp * 4,
        "k_pyramid_grey_rgb8": min(p_in, 4 * p0) * 3 + sp * 4,
        # kw in {7, 13}: blur + |DoG| + extrema of the tile interiors in one pass; |DoG| is a fused
        # temporary.  The seam test (k_extrema_seams) re-reads levels around the few tile-perimeter
        # pixels above the colour threshold, which is not compulsory traffic: it has no bytes of its
        # own and is counted here.
        "k_blur_extrema": sp * 4 * (1 + (ns - 1)),           # read grey, write 6 levels
        # the split pipeline with |DoG| planes through HBM, the traffic k_blur_extrema replaces
        # (the generic windows run k_blur_dog_generic + k_extrema_scan over every pixel)
        "k_blur_dog": sp * 4 * (1 + 2 * (ns - 1)),            # read grey, write 6 levels + 6 |DoG|
        "k_extrema_scan": sp * 4 * (ns - 1),                  # reads the |DoG| levels once
        "k_rank_sort": n_desc * 8,
        "k_refine": n_desc * (27 * 4 + 40),
        "k_orientation": n_desc * (196 * 4 + 8),
        "k_expand_scan": n_desc * 16,
        "k_descriptor": n_desc * (16 + 512),                  # §8d: outputs n_kp*(16+512)
        "k_match_decide": n_desc * 32,
        "k_linear_blend": roi * 12 + tw * th * 12,
        "k_mb_first_level": roi * (12 + 16),
        "k_mb_weight_argmax": roi * 8,
        "k_mb_blur": roi * 32,                                # read + write one float4 level (both passes fused)
        "k_mb_accumulate": roi * (16 + 12) + tw * th * 12,
        "k_fill": tw * th * 12,
        "k_crop_masks": tw * th * 12,
        "k_f32_to_rgb8": tw * th * 15,
    }


def kernel_table(prof, prof_steps, ab, flops, hbm_peak, tf_peak):
    """prof: name -> (launches, total ms) over prof_steps steps."""
    kernels = {}
    tot = sum(v[1] for v in prof.values())
    for name, (cnt, tms) in sorted(prof.items(), key=lambda kv: -kv[1][1]):
        per_step = tms / prof_steps
        ent = {"launches_per_step": cnt / prof_steps, "ms_per_step": per_step, "share": tms / tot if tot else 0}
        if name == "k_tc_top2" and flops:
            ent.update(bound="tensor", achieved=flops / (per_step * 1e-3) / 1e12, peak=tf_peak, unit="TFLOP/s")
        elif ab.get(name):
            ent.update(bound="hbm", achieved=ab[name] / (per_step * 1e-3) / 1e9, peak=hbm_peak, unit="GB/s")
        if "achieved" in ent:
            ent["frac"] = ent["achieved"] / ent["peak"]
        kernels[name] = ent
    return kernels


def top_roofline(kernels, peak_src):
    if not kernels:
        return None
    top = max(kernels, key=lambda k: kernels[k]["share"])
    t = kernels[top]
    return {"kernel": top, "bound": t.get("bound"), "achieved": t.get("achieved"), "peak": t.get("peak"),
            "unit": t.get("unit"), "frac": t.get("frac"), "traffic": None, "peak_source": peak_src,
            "share_of_step": t["share"], "ms_per_step": t["ms_per_step"]}


def load_peaks():
    import json
    pk = ROOT / "MEASURED_PEAKS.json"
    if pk.exists():
        p = json.loads(pk.read_text())
        return float(p.get("hbm_gbs", 3350.0)), float(p.get("bf16_tflops_sustained", p.get("bf16_tflops", 989.0))), "measured"
    return 3350.0, 989.0, "H100 SXM data sheet (700 W)"


# ----------------------------------------------------------------------------- inputs
def quantise(views, threads=None):
    """8-bit pixels as the reference decodes them (CImg<unsigned char>, imgio.cc:72)."""
    threads = threads or max(1, min(32, len(os.sched_getaffinity(0))))
    with ThreadPoolExecutor(threads) as ex:
        return list(ex.map(lambda v: (v * 255.0 + 0.5).astype(np.uint8), views))


def read_img_f32(pix):
    """read_img's conversion on the host (imgio.cc:79-81): (float)((double)v / 255.0)."""
    return (pix.astype(np.float32).astype(np.float64) / 255.0).astype(np.float32)


class Timer:
    """CUDA-event timing on the engine's stream (torch's current stream)."""

    def __init__(self):
        import torch
        self.torch = torch

    def ms(self, fn):
        t = self.torch
        e0, e1 = t.cuda.Event(enable_timing=True), t.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)


def silence_stdout(fn):
    """The reference prints its timers on stdout; keep fd 1 clean while it runs."""
    sys.stdout.flush()
    devnull = os.open(os.devnull, os.O_WRONLY)
    saved = os.dup(1)
    os.dup2(devnull, 1)
    try:
        return fn()
    finally:
        os.dup2(saved, 1)
        os.close(devnull)
        os.close(saved)


# ----------------------------------------------------------------------------- one stack config
def run_stack(eng, label, cfg_name, pairs_fn, bands, params, steps=5, max_output=None, n=None, cpu_views=None,
              cpu_loader=None, all_cpus=None):
    import torch
    from openpano_b200 import synth

    hbm_peak, tf_peak, peak_src = load_peaks()
    tm = Timer()
    t0 = time.perf_counter()
    views, org = synth.config_stack(cfg_name, n=n)
    h, w = views[0].shape[:2]
    pix = quantise(views)
    del views
    gen_s = time.perf_counter() - t0
    nimg = len(pix)
    items, geom = synth.translation_blend_setup(org, w, h, max_output)
    pairs = pairs_fn(nimg)
    shapes = [(h, w)] * nimg
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    mpx = nimg * h * w / 1e6

    # device buffers: 8-bit sources, f32 images, f32 mosaic, packed 8-bit mosaic (+ crop rectangle)
    px_b, im_b = (h * w * 3 + 255) // 256 * 256, (h * w * 12 + 255) // 256 * 256
    d_pix = eng.dev_alloc(px_b * nimg)
    d_img = eng.dev_alloc(im_b * nimg)
    d_out = eng.dev_alloc(ow * oh * 12)
    d_out8 = eng.dev_alloc(256 + ow * oh * 3)
    pix_ptrs = [d_pix + k * px_b for k in range(nimg)]
    img_ptrs = [d_img + k * im_b for k in range(nimg)]
    host_pix = [torch.from_numpy(p).pin_memory() for p in pix]
    host_out8 = torch.empty(256 + ow * oh * 3, dtype=torch.uint8).pin_memory()
    ws, hs = [w] * nimg, [h] * nimg

    def upload():
        for t, dp in zip(host_pix, pix_ptrs):
            eng.dev_upload_async(dp, t.data_ptr(), h * w * 3)

    def convert():
        eng.rgb8_to_mat32f_batch_dev(pix_ptrs, ws, hs, [3] * nimg, img_ptrs)

    def step_device():
        fs = eng.sift_detect_batch_ptr(img_ptrs, ws, hs, params, device=True)
        tot = eng.match_pairs_dev(fs, pairs, params)
        eng.blend_dev(img_ptrs, shapes, items, geom, d_out, ow, oh, bands, params)
        fs.free()
        return tot

    def job_e2e():
        upload()
        convert()
        fs = eng.sift_detect_batch_ptr(img_ptrs, ws, hs, params, device=True)
        m = eng.match_pairs(fs, pairs, params)
        eng.blend_dev(img_ptrs, shapes, items, geom, d_out, ow, oh, bands, params)
        eng.crop_rect_dev(d_out, ow, oh, d_out8)
        eng.mat32f_to_rgb8_dev(d_out, ow, oh, d_out8, d_out8 + 256)
        eng.dev_download_async(host_out8.data_ptr(), d_out8, 256 + ow * oh * 3)
        eng.sync()
        fs.free()
        return m

    upload()
    convert()
    eng.sync()
    # counts + untimed warm-up (allocator pool, function attributes)
    fs = eng.sift_detect_batch_ptr(img_ptrs, ws, hs, params, device=True)
    counts = [fs.count(i) for i in range(nimg)]
    d0 = fs.download(0)
    first_pair = pairs[0]
    da, db = fs.download(first_pair[0])[1], fs.download(first_pair[1])[1]
    m0 = eng.match_pairs(fs, [first_pair], params)[0]
    fs.free()
    n_matches = step_device()
    step_device()
    dev_ms = sorted(tm.ms(step_device) for _ in range(steps))
    ms_device = dev_ms[len(dev_ms) // 2]

    job_e2e()
    e2e = []
    for _ in range(3):
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        job_e2e()
        e2e.append((time.perf_counter() - t1) * 1e3)
    e2e_ms = sorted(e2e)[1]
    rect = host_out8[:16].numpy().view(np.int32)
    crop_ok = bool(rect[2] > 0 and rect[3] > 0)

    # per-kernel times of one step
    eng.profile(True)
    eng.profile_reset()
    step_device()
    prof = eng.profile_read()
    eng.profile(False)
    flops = sum(2.0 * counts[i] * counts[j] * 128 for i, j in pairs)
    kernels = kernel_table(prof, 1, algorithmic_bytes(shapes, items, params, counts, bands), flops, hbm_peak, tf_peak)

    # bounded parity sample against the oracle port
    parity = None
    try:
        from tests.checker import get_checker
        orc = get_checker("orc")
        co, do = orc.sift_detect(read_img_f32(pix[0]), params)
        mt = get_checker("orc_mt")
        parity = {"features_image0": bool(np.array_equal(co.view(np.uint64), d0[0].view(np.uint64)) and
                                          np.array_equal(do.view(np.uint32), d0[1].view(np.uint32))),
                  "matches_pair0": bool(np.array_equal(m0, mt.match(da, db, params))),
                  "against": "oracle port (oracle/liboracle.so), bit-exact comparison"}
    except Exception as ex:  # the checker is optional equipment on the box
        parity = {"unavailable": repr(ex)}

    # CPU baseline: the reference's own TUs on a bounded sample of the same stack
    cpu = None
    if cpu_loader is not None:
        try:
            if all_cpus:
                os.sched_setaffinity(0, all_cpus)
            chk, kind = cpu_loader()
            k = nimg if cpu_views is None else min(cpu_views, nimg)
            sub_imgs = [read_img_f32(p) for p in pix[:k]]
            sub_items, sub_geom = synth.translation_blend_setup(org[:k], w, h, max_output)
            sub_pairs = [pq for pq in pairs if pq[0] < k and pq[1] < k]
            p_cpu = params
            t1 = time.perf_counter()
            nf, nm, _, secs = silence_stdout(lambda: chk.hotpath(sub_imgs, sub_pairs, sub_items, sub_geom, bands, p_cpu,
                                                                 use_flann=True))
            dt = time.perf_counter() - t1
            cpu = {"value": k * h * w / 1e6 / dt, "unit": "Mpx/s", "cores": chk.num_threads(), "kind": kind,
                   "sample": f"{k} of {nimg} views, {len(sub_pairs)} pairs, one pass ({dt:.2f} s)",
                   "stage_ms": {"features": secs[0] * 1e3, "match": secs[1] * 1e3, "blend": secs[2] * 1e3}}
            del sub_imgs
        except Exception as ex:
            cpu = {"value": None, "unit": "Mpx/s", "cores": 0, "kind": "unavailable", "sample": repr(ex)}

    for p_ in (d_pix, d_img, d_out, d_out8):
        eng.dev_free(p_)
    eng.sync()
    res = {"workload": label, "images": nimg, "image_wh": [w, h], "pairs": len(pairs), "bands": bands,
           "canvas_wh": [ow, oh], "input_mpx": mpx, "gen_s": round(gen_s, 1),
           "ms_device": ms_device, "value": mpx / (ms_device * 1e-3), "unit": "Mpx/s",
           "e2e": {"ms": e2e_ms, "value": mpx / (e2e_ms * 1e-3), "unit": "Mpx/s",
                   "h2d_bytes": nimg * h * w * 3, "d2h_bytes": 256 + ow * oh * 3 + int(n_matches) * 8,
                   "boundary": "rgb8 in, cropped rgb8 mosaic + match lists out, one job at a time", "crop_ok": crop_ok},
           "features": int(sum(counts)), "matches": int(n_matches), "match_rows_rescanned_exactly": eng.match_last_exact_rows(),
           "match_rows_nominated_on_request": eng.match_last_nominated_rows(),
           "roofline": top_roofline(kernels, peak_src),
           "kernels": {k: v for k, v in list(kernels.items())[:8]},
           "parity_sample": parity, "cpu_baseline": cpu}
    return res


# ----------------------------------------------------------------------------- config 1: cylinder mode
def run_cylinder(eng, label, cfg_name, params, steps=20, cpu_loader=None, all_cpus=None):
    """BASELINE config 1 (CMU0, cylinder mode): the hot-path stages CylinderStitcher::build chains
    (cylstitcher.cc:20-87) at that shape, device-resident — SIFT, the adjacent-pair matches, the batched
    cylinder warp of every image (pano_cyl_warp_batch_dev) and the LinearBlender composite of the warped
    images with generator-known translations.  The geometry between the stages (update_h_factor, RANSAC,
    perspective_correction) is host code outside the path and not timed."""
    from openpano_b200 import synth

    hbm_peak, tf_peak, peak_src = load_peaks()
    tm = Timer()
    views, org = synth.config_stack(cfg_name)
    h, w = views[0].shape[:2]
    pix = quantise(views)
    del views
    imgs = [read_img_f32(p_) for p_ in pix]
    n = len(imgs)
    mpx = n * h * w / 1e6
    ow, oh, _, _ = eng.cyl_warp_shape(w, h, 1.0, params)
    items, geom = synth.translation_blend_setup(org, ow, oh)
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    pairs = [(k, k + 1) for k in range(n - 1)]
    shapes, wshapes = [(h, w)] * n, [(oh, ow)] * n
    d_img = [eng.dev_alloc(h * w * 12) for _ in range(n)]
    d_warp = [eng.dev_alloc(oh * ow * 12) for _ in range(n)]
    d_out = eng.dev_alloc(tw * th * 12)
    for d, im in zip(d_img, imgs):
        eng.dev_upload(d, im)
    ws, hs = [w] * n, [h] * n

    def step_device():
        fs = eng.sift_detect_batch_ptr(d_img, ws, hs, params, device=True)
        tot = eng.match_pairs_dev(fs, pairs, params)
        eng.cyl_warp_batch_dev(d_img, shapes, d_warp, None, 1.0, params)
        eng.blend_dev(d_warp, wshapes, items, geom, d_out, tw, th, 0, params)
        fs.free()
        return tot

    fs = eng.sift_detect_batch_ptr(d_img, ws, hs, params, device=True)
    counts = [fs.count(i) for i in range(n)]
    d0 = fs.download(0)
    fs.free()
    n_matches = step_device()
    step_device()
    dev_ms = sorted(tm.ms(step_device) for _ in range(steps))
    ms_device = dev_ms[len(dev_ms) // 2]
    eng.profile(True)
    eng.profile_reset()
    step_device()
    prof = eng.profile_read()
    eng.profile(False)
    ab = algorithmic_bytes(shapes, items, params, counts, 0)
    ab["k_cyl_warp"] = n * (h * w + oh * ow) * 12                     # SURVEY.md 8d: 12*(P_in + P_out) per image
    ab["k_linear_blend"] = n * oh * ow * 12 + tw * th * 12
    flops = sum(2.0 * counts[i] * counts[j] * 128 for i, j in pairs)
    kernels = kernel_table(prof, 1, ab, flops, hbm_peak, tf_peak)
    warped0 = np.empty((oh, ow, 3), np.float32)
    eng.dev_download(warped0, d_warp[0])

    parity = None
    try:
        from tests.checker import get_checker
        orc = get_checker("orc")
        co, do = orc.sift_detect(imgs[0], params)
        parity = {"features_image0": bool(np.array_equal(co.view(np.uint64), d0[0].view(np.uint64)) and
                                          np.array_equal(do.view(np.uint32), d0[1].view(np.uint32))),
                  "warped_image0": bool(np.array_equal(orc.cyl_warp(imgs[0], None, 1.0, params)[0].view(np.uint32),
                                                       warped0.view(np.uint32))),
                  "against": "oracle port (oracle/liboracle.so), bit-exact comparison"}
    except Exception as ex:
        parity = {"unavailable": repr(ex)}

    cpu = None
    if cpu_loader is not None:
        try:
            if all_cpus:
                os.sched_setaffinity(0, all_cpus)
            chk, kind = cpu_loader()
            o_items, o_geom = synth.translation_blend_setup(org, w, h)
            t1 = time.perf_counter()
            nf, nm, _, secs = silence_stdout(lambda: chk.hotpath(imgs, pairs, o_items, o_geom, 0, params, use_flann=True))
            t2 = time.perf_counter()
            with ThreadPoolExecutor(n) as ex:                          # the reference warps under `omp parallel for` (cylstitcher.cc:66)
                warped = list(ex.map(lambda im: chk.cyl_warp(im, None, 1.0, params)[0], imgs))
            t3 = time.perf_counter()
            silence_stdout(lambda: chk.blend(warped, items, geom, 0, params))
            t4 = time.perf_counter()
            total = secs[0] + secs[1] + (t3 - t2) + (t4 - t3)
            cpu = {"value": mpx / total, "unit": "Mpx/s", "cores": chk.num_threads(), "kind": kind,
                   "sample": f"{n} of {n} views, {len(pairs)} pairs, one pass ({total:.2f} s; SIFT + FLANN match + "
                             "CylinderWarper::warp + LinearBlender::run on the warped images)",
                   "stage_ms": {"features": secs[0] * 1e3, "match": secs[1] * 1e3, "warp": (t3 - t2) * 1e3,
                                "blend": (t4 - t3) * 1e3}}
        except Exception as ex:
            cpu = {"value": None, "unit": "Mpx/s", "cores": 0, "kind": "unavailable", "sample": repr(ex)}

    for p_ in d_img + d_warp + [d_out]:
        eng.dev_free(p_)
    eng.sync()
    return {"workload": label, "images": n, "image_wh": [w, h], "pairs": len(pairs), "bands": 0,
            "warped_wh": [ow, oh], "canvas_wh": [tw, th], "input_mpx": mpx,
            "ms_device": ms_device, "value": mpx / (ms_device * 1e-3), "unit": "Mpx/s",
            "features": int(sum(counts)), "matches": int(n_matches),
            "roofline": top_roofline(kernels, peak_src),
            "kernels": {k: v for k, v in list(kernels.items())[:9] + [(k, v) for k, v in kernels.items() if k == "k_cyl_warp"]},
            "parity_sample": parity, "cpu_baseline": cpu}


# ----------------------------------------------------------------------------- config 4: match sweep
def sweep_sets(n, seed=4):
    from openpano_b200 import synth
    rng = np.random.RandomState(seed)
    a = synth.rootsift_like(n, seed)
    b = a[rng.permutation(n)].copy()
    half = n // 2
    b[:half] += rng.randn(half, 128).astype(np.float32) * 10.0
    b[half:] = synth.rootsift_like(n - half, seed + 1)
    return a, b


def run_sweep(eng, sizes, params, cpu_n=10000, reps=3):
    hbm_peak, tf_peak, peak_src = load_peaks()
    tm = Timer()
    out = {"workload": "descriptor brute-force match sweep, N = M, 128-D RootSIFT-like rows", "sizes": {},
           "flops_model": "2*N*M*128 per pair (one GEMM serves both directions, SURVEY.md §8d)",
           "peak_tflops": tf_peak, "peak_source": peak_src}
    for n in sizes:
        a, b = sweep_sets(n)
        fs = eng.featureset_upload([a, b])
        tot = eng.match_pairs_dev(fs, [(0, 1)], params)       # builds the fp16 operands once, warms the pool
        ms = sorted(tm.ms(lambda: eng.match_pairs_dev(fs, [(0, 1)], params)) for _ in range(reps))[reps // 2]
        eng.profile(True)
        eng.profile_reset()
        eng.match_pairs_dev(fs, [(0, 1)], params)
        prof = eng.profile_read()
        eng.profile(False)
        fs.free()
        tf = 2.0 * n * n * 128 / (ms * 1e-3) / 1e12
        gemm_ms = prof.get("k_tc_top2", (0, 0.0))[1]
        out["sizes"][str(n)] = {"ms": ms, "matches": int(tot), "tflops_algorithmic": tf, "frac_of_peak": tf / tf_peak,
                                "k_tc_top2_ms": gemm_ms,
                                "k_tc_top2_tflops_algorithmic": (2.0 * n * n * 128 / (gemm_ms * 1e-3) / 1e12) if gemm_ms else None,
                                "rows_rescanned_exactly": eng.match_last_exact_rows(),
                                "rows_nominated_on_request": eng.match_last_nominated_rows()}
        del a, b
    try:
        from tests.checker import get_checker, have
        chk = get_checker("ref" if have("ref") else "orc")
        a, b = sweep_sets(cpu_n)
        t1 = time.perf_counter()
        m = chk.match(a, b, params)
        dt = time.perf_counter() - t1
        got = eng.match_bruteforce(a, b, params)
        out["cpu_baseline"] = {"value": 2.0 * cpu_n * cpu_n * 128 / dt / 1e12, "unit": "TFLOP/s", "cores": 1,
                               "kind": "reference" if have("ref") else "port",
                               "sample": f"FeatureMatcher::match (matcher.cc:15-71) on {cpu_n} x {cpu_n} rows, {dt:.2f} s",
                               "pairs_identical_to_gpu": bool(np.array_equal(m, got))}
    except Exception as ex:
        out["cpu_baseline"] = {"value": None, "unit": "TFLOP/s", "cores": 0, "kind": "unavailable", "sample": repr(ex)}
    return out


# ----------------------------------------------------------------------------- sharded leg (N > 1)
def run_sharded(eng, rank, world, params, cfg_name="unordered_38x1300x867", bands=0, reps=5):
    """Config 3 sharded across the ranks by DistributedStitcher (images k mod G -> C1 descriptor
    all-gather -> dealt pair tasks -> strip blend -> C2 strip gather), timed on the device as the
    max over ranks; rank 0 then repeats the job alone and compares bit for bit."""
    import torch
    import torch.distributed as dist
    from openpano_b200 import synth
    from openpano_b200.parallel import DistributedStitcher, shard_images

    views, org = synth.config_stack(cfg_name)
    pix = quantise(views)
    del views
    n = len(pix)
    h, w = pix[0].shape[:2]
    items, geom = synth.translation_blend_setup(org, w, h)
    pairs = synth.all_pairs(n)
    shapes = [(h, w)] * n
    mine = shard_images(n, world, rank)
    owned_pix = {k: torch.from_numpy(pix[k]).cuda() for k in mine}
    ds = DistributedStitcher(eng, params)
    best = None
    for rep in range(reps + 1):
        torch.cuda.synchronize()
        dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        matches, mosaic = ds.run_rgb8(owned_pix, n, shapes, pairs, items, geom, bands)
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rep > 0 and (best is None or t.item() < best[0]):
            phases = torch.tensor([ds.ms.get(k, 0.0) for k in ds.PHASES], device="cuda")
            dist.all_reduce(phases, op=dist.ReduceOp.MAX)
            best = (t.item(), dict(zip(ds.PHASES, [float(x) for x in phases.tolist()])), dict(ds.host_ms))
    res = None
    if rank == 0:
        all_pix = [torch.from_numpy(p).cuda() for p in pix]
        all_img = [torch.empty((h, w, 3), dtype=torch.float32, device="cuda") for _ in pix]
        ptrs = [t_.data_ptr() for t_ in all_img]
        tw, th = max(it[2] for it in items), max(it[3] for it in items)
        ref_out = torch.empty((th, tw, 3), dtype=torch.float32, device="cuda")
        one = []
        for rep in range(3):
            torch.cuda.synchronize()
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            eng.rgb8_to_mat32f_batch_dev([t_.data_ptr() for t_ in all_pix], [w] * n, [h] * n, [3] * n, ptrs)
            fs = eng.sift_detect_batch_ptr(ptrs, [w] * n, [h] * n, params, device=True)
            ref_m = eng.match_pairs(fs, pairs, params)
            eng.blend_dev(ptrs, shapes, items, geom, ref_out.data_ptr(), tw, th, bands, params)
            s1.record()
            torch.cuda.synchronize()
            fs.free()
            one.append(s0.elapsed_time(s1))
        one_ms = min(one[1:])
        same_m = len(matches) == len(ref_m) and all(np.array_equal(a, b) for a, b in zip(matches, ref_m))
        same_o = bool(torch.equal(mosaic, ref_out))
        mpx = n * h * w / 1e6
        limiting = max(best[1], key=best[1].get)
        res = {"workload": f"{cfg_name}: {n} images, {len(pairs)} pairs, bands {bands}", "n_gpus": world,
               "partition": "images k mod G -> C1 all-gather(descriptors) -> pairs dealt by N_i*N_j -> canvas row strips -> C2 all-gather(strips)",
               "ms_sharded": best[0], "phase_ms_max_over_ranks": best[1], "phase_host_ms_rank0": best[2],
               "limiting_phase": limiting,
               "ms_one_gpu": one_ms, "efficiency_vs_one_gpu": one_ms / (world * best[0]),
               "speedup_vs_one_gpu": one_ms / best[0], "value": mpx / (best[0] * 1e-3), "unit": "Mpx/s",
               "matches": int(sum(len(m) for m in matches)), "matches_identical": bool(same_m),
               "mosaic_identical": same_o}
    dist.barrier()
    return res


def run_sharded_sweep(eng, rank, world, params, n=100000, reps=3):
    """Config 4 row-sharded across the ranks: every rank holds both descriptor sets and decides its
    contiguous share of the smaller set's rows (pano_match_pairs_shard: the reference's `parallel for`
    over k, matcher.cc:32); no collective on the data path.  Timed on the device as the max over
    ranks; rank 0 repeats the match alone and compares the concatenated lists pair for pair."""
    import torch
    import torch.distributed as dist

    a, b = sweep_sets(n)
    fs = eng.featureset_upload([a, b])
    del a, b
    eng.match_pairs_dev(fs, [(0, 1)], params, shard=(rank, world))       # fp16 operands + pool warm-up
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.match_pairs_dev(fs, [(0, 1)], params, shard=(rank, world))
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        times.append(float(t.item()))
    mine = eng.match_pairs(fs, [(0, 1)], params, shard=(rank, world))[0]
    gathered = [None] * world
    dist.all_gather_object(gathered, mine)
    res = None
    if rank == 0:
        one = []
        for _ in range(reps):
            torch.cuda.synchronize()
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            eng.match_pairs_dev(fs, [(0, 1)], params)
            s1.record()
            torch.cuda.synchronize()
            one.append(s0.elapsed_time(s1))
        full = eng.match_pairs(fs, [(0, 1)], params)[0]
        cat = np.concatenate(gathered) if gathered else np.zeros((0, 2), np.int32)
        ms, one_ms = sorted(times)[len(times) // 2], sorted(one)[len(one) // 2]
        _, tf_peak, _ = load_peaks()
        tf = 2.0 * n * n * 128 / (ms * 1e-3) / 1e12
        res = {"workload": f"descriptor brute-force match, {n} x {n} rows, rows of the smaller set split over the ranks",
               "n_gpus": world, "partition": "rank r decides rows [n*r/G, n*(r+1)/G) of the smaller set against all rows; no data-path collective",
               "ms_sharded": ms, "ms_one_gpu": one_ms, "speedup_vs_one_gpu": one_ms / ms, "efficiency_vs_one_gpu": one_ms / (world * ms),
               "tflops_algorithmic": tf, "frac_of_peak_all_gpus": tf / (tf_peak * world), "matches": int(len(full)),
               "pairs_identical": bool(np.array_equal(cat, full))}
    fs.free()
    dist.barrier()
    return res
