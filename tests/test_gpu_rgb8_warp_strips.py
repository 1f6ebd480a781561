"""GPU: the cylinder warp and the row strips of the composite straight from decoded 8-bit pixels
(pano_cyl_warp_batch_rgb8_dev, pano_blend_rows_rgb8_dev), without f32 copies of the source images.  Every
result must have the raw bits of the same stage on read_img's f32 images of the same pixels.  Also config 1's
cylinder chain from 8-bit pixels, the invalid calls, and the sharded stitcher's 8-bit path on two GPUs."""
import ctypes as C
import json
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests import golden_util as gu
from tests.test_gpu_match_warp_blend import _perspective_items

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent


def _pix(w, h, seed, channels):
    pix = (synth.make_canvas(h, w, seed) * 255.0 + 0.5).astype(np.uint8)
    return pix if channels == 3 else np.ascontiguousarray(pix[..., 1])


def _chans(pix):
    return [1 if x.ndim == 2 else 3 for x in pix]


def _kpts(w, h, seed, n=40):
    """Image-centred keypoints, a few of them outside the image."""
    rng = np.random.RandomState(seed)
    k = (rng.rand(n, 2) - 0.5) * np.array([w * 1.1, h * 1.1])
    return np.ascontiguousarray(k, np.float64)


class _Dev:
    """Device buffers freed together."""

    def __init__(self, engine):
        self.eng, self.ptrs = engine, []

    def alloc(self, nbytes):
        p = self.eng.dev_alloc(nbytes)
        self.ptrs.append(p)
        return p

    def upload(self, arr):
        p = self.alloc(arr.nbytes)
        self.eng.dev_upload(p, arr)
        return p

    def free(self):
        for p in self.ptrs:
            self.eng.dev_free(p)
        self.ptrs = []


def _converted(engine, dev, d_pix, pix):
    """read_img's f32 images of the pixels, on the device (pano_rgb8_to_mat32f_batch_dev)."""
    d_f32 = [dev.alloc(x.shape[0] * x.shape[1] * 12) for x in pix]
    engine.rgb8_to_mat32f_batch_dev(d_pix, [x.shape[1] for x in pix], [x.shape[0] for x in pix], _chans(pix), d_f32)
    return d_f32


# ----------------------------------------------------------------------------- cylinder warp
def _warp_both(engine, pix, hf, kpts, p=None):
    """(f32 warps of the converted images, 8-bit warps, f32-rewritten keypoints, 8-bit-rewritten keypoints)."""
    p = p or default_params()
    shapes = [x.shape[:2] for x in pix]
    outs = [engine.cyl_warp_shape(w, h, hf, p)[:2] for h, w in shapes]
    dev = _Dev(engine)
    try:
        d_pix = [dev.upload(x) for x in pix]
        d_f32 = _converted(engine, dev, d_pix, pix)
        d_a = [dev.alloc(ow * oh * 12) for ow, oh in outs]
        d_b = [dev.alloc(ow * oh * 12) for ow, oh in outs]
        ka, kb = [k.copy() for k in kpts], [k.copy() for k in kpts]
        engine.cyl_warp_batch_dev(d_f32, shapes, d_a, ka, hf, p)
        engine.cyl_warp_batch_rgb8_dev(d_pix, _chans(pix), shapes, d_b, kb, hf, p)
        want, got = [], []
        for (ow, oh), a, b in zip(outs, d_a, d_b):
            wa, gb = np.empty((oh, ow, 3), np.float32), np.empty((oh, ow, 3), np.float32)
            engine.dev_download(wa, a)
            engine.dev_download(gb, b)
            want.append(wa)
            got.append(gb)
    finally:
        dev.free()
    return want, got, ka, kb


def _check_warps(orc, pix, hf, kpts, want, got, ka, kb, p=None):
    for k, x in enumerate(pix):
        o_img, o_kp = orc.cyl_warp(orc.read_img_rgb8(x), kpts[k], hf, p)
        assert gu.same_bits(want[k], o_img), f"f32 warp of image {k}"
        assert gu.same_bits(got[k], want[k]), f"8-bit warp of image {k}"
        assert gu.same_bits(kb[k], ka[k]) and gu.same_bits(ka[k], o_kp), f"keypoints of image {k}"
        unmapped = got[k][..., 0] == -1
        assert unmapped.any() and (got[k][unmapped] == -1).all(), f"unmapped pixels of image {k}"
        assert (got[k][~unmapped] >= 0).all()


@pytest.mark.parametrize("hf", [1.0, 1.2])
@pytest.mark.parametrize("channels", [3, 1])
def test_cyl_warp_rgb8_equals_warp_of_read_img(engine, orc, channels, hf):
    w, h = 333, 217                                    # neither a multiple of the 32×8 block
    pix = [_pix(w, h, 17 + channels, channels)]
    kpts = [_kpts(w, h, 3)]
    _check_warps(orc, pix, hf, kpts, *_warp_both(engine, pix, hf, kpts))


@pytest.mark.parametrize("hf", [1.0, 1.2])
def test_cyl_warp_rgb8_mixed_batch(engine, orc, hf):
    """One launch over different shapes and channel counts (a 3×3 image warps to 1×2); one image without
    keypoints."""
    shapes = [(600, 400, 3), (257, 311, 1), (130, 97, 3), (45, 64, 1), (31, 9, 3), (3, 3, 1)]
    pix = [_pix(w, h, 5 * k + 2, c) for k, (w, h, c) in enumerate(shapes)]
    kpts = [_kpts(w, h, k) for k, (w, h, _) in enumerate(shapes)]
    kpts[2] = np.zeros((0, 2), np.float64)
    _check_warps(orc, pix, hf, kpts, *_warp_both(engine, pix, hf, kpts))


# ----------------------------------------------------------------------------- config 1 from 8-bit pixels
def _features(fs):
    out = [fs.download(i) for i in range(fs.n_images)]
    fs.free()
    return out


def _cylinder_chain(engine, dev, pix, d_src, rgb8, pairs, org, p):
    """SIFT -> adjacent matches -> warp of images and keypoints -> linear composite, all on the device."""
    n, (h, w) = len(pix), pix[0].shape[:2]
    ws, hs = [w] * n, [h] * n
    if rgb8:
        fs = engine.sift_detect_batch_rgb8_ptr(d_src, ws, hs, _chans(pix), p, device=True)
    else:
        fs = engine.sift_detect_batch_ptr(d_src, ws, hs, p, device=True)
    matches = engine.match_pairs(fs, pairs, p)
    feats = _features(fs)
    ow, oh, _, _ = engine.cyl_warp_shape(w, h, 1.0, p)
    d_warp = [dev.alloc(oh * ow * 12) for _ in range(n)]
    kp = [np.ascontiguousarray(c).copy() for c, _ in feats]
    if rgb8:
        engine.cyl_warp_batch_rgb8_dev(d_src, _chans(pix), [(h, w)] * n, d_warp, kp, 1.0, p)
    else:
        engine.cyl_warp_batch_dev(d_src, [(h, w)] * n, d_warp, kp, 1.0, p)
    items, geom = synth.translation_blend_setup(org, ow, oh)
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    d_out = dev.alloc(tw * th * 12)
    engine.blend_dev(d_warp, [(oh, ow)] * n, items, geom, d_out, tw, th, 0, p)
    warped = []
    for d in d_warp:
        a = np.empty((oh, ow, 3), np.float32)
        engine.dev_download(a, d)
        warped.append(a)
    mosaic = np.empty((th, tw, 3), np.float32)
    engine.dev_download(mosaic, d_out)
    return feats, matches, warped, kp, mosaic


def test_config1_cylinder_chain_from_rgb8(engine, orc):
    """BASELINE config 1 (8 × 600×400, cylinder mode) at its shape: SIFT, the 7 adjacent-pair matches, the warp of
    every image and its keypoints and the LinearBlender composite of the warped images, read from 8-bit pixels,
    are today's f32 chain on the converted images, bit for bit."""
    views, org = synth.config_stack("cmu0_8x600x400")
    pix = [(v * 255.0 + 0.5).astype(np.uint8) for v in views]
    p = default_params(ordered_input=1)
    pairs = [(k, k + 1) for k in range(len(pix) - 1)]
    dev = _Dev(engine)
    try:
        d_pix = [dev.upload(x) for x in pix]
        d_f32 = _converted(engine, dev, d_pix, pix)
        want = _cylinder_chain(engine, dev, pix, d_f32, False, pairs, org, p)
        got = _cylinder_chain(engine, dev, pix, d_pix, True, pairs, org, p)
    finally:
        dev.free()
    (wf, wm, ww, wk, wo), (gf, gm, gw, gk, go) = want, got
    assert sum(len(d) for _, d in wf) > 3000 and sum(len(m) for m in wm) > 500
    for k, ((wc, wd), (gc, gd)) in enumerate(zip(wf, gf)):
        assert gu.same_bits(gc, wc) and gu.same_bits(gd, wd), f"features of image {k}"
    assert len(gm) == len(wm) and all(np.array_equal(a, b) for a, b in zip(gm, wm)), "match lists"
    for k in range(len(pix)):
        assert gu.same_bits(gw[k], ww[k]), f"warped image {k}"
        assert gu.same_bits(gk[k], wk[k]), f"warped keypoints of image {k}"
    assert gu.same_bits(go, wo), "mosaic"
    o_img, _ = orc.cyl_warp(orc.read_img_rgb8(pix[0]), None, 1.0, p)
    assert gu.same_bits(gw[0], o_img)


# ----------------------------------------------------------------------------- row strips
def strip_halo(bands, gauss_window_factor):
    """Rows a multiband strip reads beyond its edges: the summed half-widths of the level blurs, whose windows
    are GaussCache's (gaussian.cc:17-20) at sigma = sqrt(2 l + 1) * 4 (multiband.cc:145-151)."""
    halo = 0
    for level in range(bands - 1):
        sigma = np.float32(math.sqrt(level * 2 + 1.0) * 4)
        kw = int(math.ceil(0.3 * float(sigma / np.float32(2) - np.float32(1)) + 0.8) * gauss_window_factor)
        if kw % 2 == 0:
            kw += 1
        halo += kw // 2
    return halo


def _gap_stack(channels):
    """Two rows of three 240×180 views with 220 canvas rows between them that no image covers."""
    canvas = (synth.make_canvas(580, 540, 41) * 255.0 + 0.5).astype(np.uint8)
    org = [(x, y) for y in (0, 400) for x in (0, 150, 300)]
    pix = [np.ascontiguousarray(canvas[y:y + 180, x:x + 240]) for x, y in org]
    if channels == 1:
        pix = [np.ascontiguousarray(x[..., 1]) for x in pix]
    items, geom = synth.translation_blend_setup(org, 240, 180)
    return pix, items, geom


def _strips_both(engine, pix, items, geom, bands, p, cuts):
    """(pano_blend_dev of the converted images, pano_blend_rgb8_dev, the strips of pano_blend_rows_rgb8_dev
    between consecutive cuts)."""
    shapes = [x.shape[:2] for x in pix]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    dev = _Dev(engine)
    try:
        d_pix = [dev.upload(x) for x in pix]
        d_f32 = _converted(engine, dev, d_pix, pix)
        d_out = dev.alloc(tw * th * 12)
        f32, full = np.empty((th, tw, 3), np.float32), np.empty((th, tw, 3), np.float32)
        engine.blend_dev(d_f32, shapes, items, geom, d_out, tw, th, bands, p)
        engine.dev_download(f32, d_out)
        engine.blend_rgb8_dev(d_pix, _chans(pix), shapes, items, geom, d_out, tw, th, bands, p)
        engine.dev_download(full, d_out)
        parts = []
        for r0, r1 in zip(cuts[:-1], cuts[1:]):
            part = np.empty((r1 - r0, tw, 3), np.float32)
            engine.blend_rows_rgb8_dev(d_pix, _chans(pix), shapes, items, geom, d_out, tw, th, r0, r1, bands, p)
            engine.dev_download(part, d_out)
            parts.append(part)
    finally:
        dev.free()
    return f32, full, parts


@pytest.mark.parametrize("projection", [0, 1])
@pytest.mark.parametrize("channels", [3, 1])
@pytest.mark.parametrize("bands", [0, 1, 3, 5])
def test_blend_rows_rgb8_concatenate_to_blend_rgb8(engine, bands, channels, projection):
    p = default_params(multiband=max(bands, 1), lazy_read=0)
    if projection == 0:
        pix, items, geom = _gap_stack(channels)
        th = max(it[3] for it in items)
        cuts = [0, 7, 7, 150, 250, 330, 401, th]       # an empty strip; [250, 330) meets no image, halo included
        empty = (250, 330)
        assert all(it[3] + strip_halo(bands, 6) < empty[0] or it[1] - strip_halo(bands, 6) >= empty[1] for it in items)
    else:
        imgs, org = synth.make_stack(4, 300, 200, 100, 7)
        items, geom = _perspective_items(org, 4, projection)
        pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
        if channels == 1:
            pix = [np.ascontiguousarray(x[..., 0]) for x in pix]
        th = max(it[3] for it in items)
        cuts = [0, 33, 33, 100, 101, th]
        empty = None
    f32, full, parts = _strips_both(engine, pix, items, geom, bands, p, cuts)
    assert (full[..., 0] >= 0).mean() > 0.3
    assert gu.same_bits(full, f32)
    assert gu.same_bits(np.concatenate(parts), full)
    if empty is not None:
        assert (parts[cuts.index(empty[0])] == -1).all()


def test_blend_rows_rgb8_halo_wider_than_256_rows(engine):
    """GAUSS_WINDOW_FACTOR 12 with MULTIBAND 16: the strip halo is 288 rows.  The strip from row 450 reads the
    first row of views, whose ROI ends 270 rows above it (row 180)."""
    bands, gwf = 16, 12
    halo = strip_halo(bands, gwf)
    assert halo == 288 and halo > 256
    pix, items, geom = _gap_stack(3)
    pix[4] = np.ascontiguousarray(pix[4][..., 2])      # a grey image among colour ones
    p = default_params(multiband=bands, gauss_window_factor=gwf, lazy_read=0)
    th = max(it[3] for it in items)
    assert 256 < 450 - max(it[3] for it in items[:3]) < halo
    cuts = [0, 100, 450, th]
    f32, full, parts = _strips_both(engine, pix, items, geom, bands, p, cuts)
    assert gu.same_bits(full, f32)
    assert gu.same_bits(np.concatenate(parts), full)


# ----------------------------------------------------------------------------- invalid calls
def test_invalid_calls(engine, orc):
    from openpano_b200.capi import LIB, PanoCylJob
    pix, items, geom = _gap_stack(3)
    pix, items = pix[:3], items[:3]
    n = len(pix)
    shapes = [x.shape[:2] for x in pix]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    p = default_params()
    vp, ip = C.c_void_p, C.c_int
    ow, oh, _, _ = engine.cyl_warp_shape(240, 180, 1.0, p)

    def arr(t, vals):
        return (t * max(len(vals), 1))(*vals)

    dev = _Dev(engine)
    try:
        d_pix = [dev.upload(x) for x in pix]
        d_warp = [dev.alloc(ow * oh * 12) for _ in pix]
        d_out = dev.alloc(tw * th * 12)

        def warp(ptrs=d_pix, ch=(3, 3, 3), out=d_warp, ws=(240,) * 3, hs=(180,) * 3, osize=(ow, oh), count=n,
                 ctx=True, jobs=True):
            js = (PanoCylJob * n)()
            for k in range(n):
                js[k].w, js[k].h, js[k].d_out_hwc = ws[k], hs[k], out[k]
                js[k].out_w, js[k].out_h = osize
            return LIB.pano_cyl_warp_batch_rgb8_dev(engine._h if ctx else None, count, js if jobs else None,
                                                    arr(vp, ptrs) if ptrs is not None else None,
                                                    arr(ip, ch) if ch is not None else None, 1.0, C.byref(p))
        assert warp() == 0
        assert warp(ctx=False) == -2
        assert warp(jobs=False) == -2
        assert warp(ptrs=None) == -2
        assert warp(ch=None) == -2
        assert warp(ptrs=[d_pix[0], None, d_pix[2]]) == -2
        assert warp(out=[d_warp[0], d_warp[1], None]) == -2
        for bad in (0, 2, 4):
            assert warp(ch=(3, bad, 3)) == -2
        assert warp(ws=(240, 1, 240)) == -2
        assert warp(hs=(180, 180, 1)) == -2
        assert warp(osize=(ow + 1, oh)) == -2
        assert warp(osize=(ow, oh - 1)) == -2

        blend_args, g = engine._blend_args([None] * n, shapes, items, geom)

        def rows(ptrs=d_pix, ch=(3, 3, 3), imgs=blend_args, geo=True, out=d_out, size=(tw, th), r=(0, th), count=n):
            return LIB.pano_blend_rows_rgb8_dev(engine._h, count, imgs, arr(vp, ptrs) if ptrs is not None else None,
                                                arr(ip, ch) if ch is not None else None, C.byref(g) if geo else None,
                                                3, C.byref(p), vp(out), size[0], size[1], r[0], r[1])
        assert rows() == 0
        assert rows(count=0) == -2
        assert rows(ptrs=None) == -2
        assert rows(ch=None) == -2
        assert rows(imgs=None) == -2
        assert rows(geo=False) == -2
        assert rows(out=None) == -2
        assert rows(ptrs=[d_pix[0], None, d_pix[2]]) == -2
        assert rows(ptrs=[d_pix[0], None, d_pix[2]], r=(0, 10)) == -2       # checked even where the strip cannot reach
        for bad in (0, 2, 4):
            assert rows(ch=(3, 3, bad)) == -2
        assert rows(size=(tw + 1, th)) == -2
        assert rows(size=(tw, th - 1)) == -2
        assert rows(r=(-1, 10)) == -2
        assert rows(r=(10, th + 1)) == -2
        assert rows(r=(20, 10)) == -2
        small, _ = engine._blend_args([None] * n, [(1, 240)] + shapes[1:], items, geom)
        assert rows(imgs=small) == -2
    finally:
        dev.free()
    # the context is still usable
    kpts = [_kpts(240, 180, k) for k in range(n)]
    _check_warps(orc, pix, 1.0, kpts, *_warp_both(engine, pix, 1.0, kpts))
    f32, full, parts = _strips_both(engine, pix, items, geom, 3, default_params(multiband=3), [0, 61, th])
    assert gu.same_bits(full, f32) and gu.same_bits(np.concatenate(parts), full)


# ----------------------------------------------------------------------------- two GPUs
@pytest.mark.parametrize("bands,extra", [(0, ()), (3, ()), (16, ("gauss_window_factor=12",))])
def test_two_rank_rgb8_equals_one_gpu(bands, extra):
    """DistributedStitcher.run_rgb8 over NCCL (SIFT and the strip read the 8-bit pixels, a grey image among
    colour ones) against the one-GPU chain on the same pixels; the last case has a 288-row strip halo."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(29531 + bands), str(ROOT / "tools" / "run_dist.py"), "small", "2",
           str(bands), "rgb8", *extra]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    res = json.loads([line for line in out.stdout.splitlines() if line.startswith("{")][-1])
    assert res["rgb8"] and res["matches_identical"] and res["mosaic_identical"], res
