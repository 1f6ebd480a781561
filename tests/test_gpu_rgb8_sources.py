"""GPU: SIFT and the blend straight from decoded 8-bit pixels (pano_sift_detect_batch_rgb8[_dev], pano_blend_rgb8_dev),
without f32 copies of the source images.  Every result must have the raw bits of the same stage on read_img's f32
images of the same pixels: the 8-bit kernels convert each tap as read_img converts it.  Also the pipelined stitcher's
8-bit path (output and device-memory high-water mark), the invalid calls and the C++ adaptor next to the reference's
read_img + SIFTDetector."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests import golden_util as gu
from tests.test_gpu_match_warp_blend import _perspective_items

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "rgb8_sift_test"
SHAPES = [(600, 400), (1300, 867), (1500, 1112), (4000, 3000), (333, 517)]   # (w, h): 600×400 is upsampled


def _pix(w, h, seed, channels):
    pix = (synth.make_canvas(h, w, seed) * 255.0 + 0.5).astype(np.uint8)
    return pix if channels == 3 else np.ascontiguousarray(pix[..., 1])


def _features(fs):
    """Per image (coordinates, real coordinates, descriptors) of a featureset."""
    from openpano_b200.capi import LIB
    out = []
    for i in range(fs.n_images):
        coor, desc = fs.download(i)
        real = np.zeros_like(coor)
        if len(coor):
            fs.eng._check(LIB.pano_featureset_download_real(fs._h, i, real.ctypes.data_as(C.POINTER(C.c_double))))
        out.append((coor, real, desc))
    fs.free()
    return out


def _same_features(a, b):
    return len(a) == len(b) and all(gu.same_bits(x, y) for fa, fb in zip(a, b) for x, y in zip(fa, fb))


def _all_entries(engine, pix, kinds=("pageable", "pinned", "device")):
    """The features of every 8-bit entry: host pageable, host pinned and device sources."""
    from openpano_b200.capi import Engine
    ws, hs = [x.shape[1] for x in pix], [x.shape[0] for x in pix]
    chans = [1 if x.ndim == 2 else x.shape[2] for x in pix]
    got = {}
    if "pageable" in kinds:
        got["pageable"] = _features(engine.sift_detect_batch_rgb8(pix))
    h_pix = [Engine.host_alloc(x.nbytes) for x in pix]
    d_pix = [engine.dev_alloc(x.nbytes) for x in pix]
    try:
        for h, d, x in zip(h_pix, d_pix, pix):
            C.memmove(h, x.ctypes.data, x.nbytes)
            engine.dev_upload(d, x)
        if "pinned" in kinds:
            got["pinned"] = _features(engine.sift_detect_batch_rgb8_ptr(h_pix, ws, hs, chans))
        if "device" in kinds:
            got["device"] = _features(engine.sift_detect_batch_rgb8_ptr(d_pix, ws, hs, chans, device=True))
    finally:
        for h in h_pix:
            Engine.host_free(h)
        for d in d_pix:
            engine.dev_free(d)
    return got


@pytest.mark.parametrize("channels", [3, 1])
@pytest.mark.parametrize("w,h", SHAPES)
def test_sift_rgb8_equals_sift_of_read_img(engine, orc, w, h, channels):
    pix = _pix(w, h, w + h, channels)
    f32 = orc.read_img_rgb8(pix)
    want = _features(engine.sift_detect_batch([f32]))
    assert len(want[0][0]) > 100
    co, do = orc.sift_detect(f32)
    assert gu.same_bits(want[0][0], co) and gu.same_bits(want[0][2], do)
    for kind, got in _all_entries(engine, [pix]).items():
        assert _same_features(got, want), kind


def test_sift_rgb8_mixed_batch(engine, orc):
    """One batch of different shapes and channel counts."""
    pix = [_pix(w, h, 7 * k + 1, 3 if k % 2 == 0 else 1) for k, (w, h) in enumerate(SHAPES)]
    pix.append(_pix(640, 480, 99, 3)[..., :1].copy())          # H×W×1 through the numpy binding
    want = _features(engine.sift_detect_batch([orc.read_img_rgb8(x) for x in pix]))
    for kind, got in _all_entries(engine, pix).items():
        assert _same_features(got, want), kind


def test_sift_rgb8_capacity_growth(monkeypatch, orc):
    """Lists that start at 256 entries grow at the first count query; the 8-bit sources are read again.  A context
    keeps the grown capacity, so every entry runs on a fresh one."""
    from openpano_b200.capi import Engine
    pix = [_pix(1300, 867, 5, 3), _pix(600, 400, 6, 1)]
    monkeypatch.delenv("PANO_SIFT_CAP", raising=False)
    eng = Engine(0)
    try:
        want = _features(eng.sift_detect_batch([orc.read_img_rgb8(x) for x in pix]))
    finally:
        eng.close()
    assert max(len(f[0]) for f in want) > 256
    monkeypatch.setenv("PANO_SIFT_CAP", "256")
    for kind in ("pageable", "pinned", "device"):
        eng = Engine(0)
        try:
            got = _all_entries(eng, pix, (kind,))[kind]
        finally:
            eng.close()
        assert _same_features(got, want), kind


def _blend_both(engine, pix, items, geom, bands, p):
    """(pano_blend_dev of the converted images, pano_blend_rgb8_dev of the pixels)."""
    shapes = [x.shape[:2] for x in pix]
    chans = [1 if x.ndim == 2 else 3 for x in pix]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    d_pix = [engine.dev_alloc(x.nbytes) for x in pix]
    d_f32 = [engine.dev_alloc(x.shape[0] * x.shape[1] * 12) for x in pix]
    d_out = engine.dev_alloc(tw * th * 12)
    want, got = np.empty((th, tw, 3), np.float32), np.empty((th, tw, 3), np.float32)
    try:
        for d, x in zip(d_pix, pix):
            engine.dev_upload(d, x)
        engine.rgb8_to_mat32f_batch_dev(d_pix, [s[1] for s in shapes], [s[0] for s in shapes], chans, d_f32)
        engine.blend_dev(d_f32, shapes, items, geom, d_out, tw, th, bands, p)
        engine.dev_download(want, d_out)
        engine.blend_rgb8_dev(d_pix, chans, shapes, items, geom, d_out, tw, th, bands, p)
        engine.dev_download(got, d_out)
    finally:
        for d in d_pix + d_f32 + [d_out]:
            engine.dev_free(d)
    return want, got


def _stack_pix(n=6, channels=3):
    imgs, org = synth.make_stack(n, 240, 180, 70, 29, rows=2, step_y=60)
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    if channels == 1:
        pix = [np.ascontiguousarray(x[..., 1]) for x in pix]
    items, geom = synth.translation_blend_setup(org, 240, 180)
    return pix, items, geom


@pytest.mark.parametrize("lazy,ordered", [(1, 0), (1, 1), (0, 0), (0, 1)])
@pytest.mark.parametrize("channels", [3, 1])
def test_linear_blend_rgb8(engine, orc, lazy, ordered, channels):
    pix, items, geom = _stack_pix(6, channels)
    p = default_params(lazy_read=lazy, ordered_input=ordered)
    want, got = _blend_both(engine, pix, items, geom, 0, p)
    assert (want[..., 0] == -1).any() and (want[..., 0] >= 0).mean() > 0.5
    assert gu.same_bits(want, orc.blend([orc.read_img_rgb8(x) for x in pix], items, geom, 0, p))
    assert gu.same_bits(got, want)


@pytest.mark.parametrize("bands", [1, 3, 5])
@pytest.mark.parametrize("channels", [3, 1])
def test_multiband_blend_rgb8(engine, bands, channels):
    pix, items, geom = _stack_pix(7, channels)
    want, got = _blend_both(engine, pix, items, geom, bands, default_params())
    assert gu.same_bits(got, want)


@pytest.mark.parametrize("projection", [0, 1, 2])
@pytest.mark.parametrize("bands", [0, 3])
def test_blend_rgb8_projections(engine, orc, projection, bands):
    imgs, org = synth.make_stack(4, 300, 200, 100, 7)
    items, geom = _perspective_items(org, 4, projection)
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    pix[1] = np.ascontiguousarray(pix[1][..., 0])               # a grey image among colour ones
    want, got = _blend_both(engine, pix, items, geom, bands, default_params())
    assert (want < 0).mean() < 0.9
    assert gu.same_bits(want, orc.blend([orc.read_img_rgb8(x) for x in pix], items, geom, bands))
    assert gu.same_bits(got, want)


def _pipelined_job(pix, pairs, items, geom, p, convert_first):
    """One PipelinedStitcher(rgb8=True) job; returns (compute-context high-water mark, output bytes, matches).
    convert_first: the stitcher's former compute path instead of run() — a per-slot f32 image block, the conversion
    launch, SIFT and the blend on the f32 copies — with the same slot buffers, streams and events."""
    from openpano_b200.stitcher import PipelinedStitcher
    shapes = [x.shape[:2] for x in pix]
    ws, hs, n = [s[1] for s in shapes], [s[0] for s in shapes], len(pix)
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    ps = PipelinedStitcher(0, p, depth=2, rgb8=True, crop=True)
    d_f32 = None
    try:
        ps.cmp.sync()
        ps.cmp.mem_high_water(reset=True)
        out = np.zeros(ps.out_bytes((ow, oh)), np.uint8)
        k = ps.stage([a.ctypes.data for a in pix], shapes, (ow, oh))
        if not convert_first:
            matches = ps.wait(ps.run(k, pairs, items, geom, out.ctypes.data))
        else:
            s = ps.slots[k]
            d_f32 = ps.cmp.dev_alloc(sum(x.nbytes * 4 for x in pix))
            ptrs = [d_f32 + 4 * sum(x.nbytes for x in pix[:q]) for q in range(n)]
            ps.cmp.event_wait(s["ev_up"])
            ps.cmp.rgb8_to_mat32f_batch_dev([s["pix"] + o for o in s["pix_offs"]], ws, hs, [3] * n, ptrs)
            fs = ps.cmp.sift_detect_batch_ptr(ptrs, ws, hs, p, device=True)
            m = ps.cmp.match_pairs(fs, pairs, p)
            ps.cmp.blend_dev(ptrs, shapes, items, geom, s["out"], ow, oh, 0, p)
            ps.cmp.crop_rect_dev(s["out"], ow, oh, s["out8"])
            ps.cmp.mat32f_to_rgb8_dev(s["out"], ow, oh, s["out8"], s["out8"] + ps.RGB8_HEADER)
            ps.cmp.event_record(s["ev_cmp"])
            fs.free()
            ps.dn.event_wait(s["ev_cmp"])
            ps.dn.dev_download_async(out.ctypes.data, s["out8"], ps.out_bytes((ow, oh)))
            ps.dn.event_record(s["ev_dn"])
            s["busy"] = True
            matches = ps.wait((k, m))
        ps.cmp.sync()
        return ps.cmp.mem_high_water(), out, matches
    finally:
        if d_f32:
            ps.cmp.dev_free(d_f32)
        ps.close()


def test_pipelined_stitcher_rgb8_reads_pixels(monkeypatch, orc):
    """PipelinedStitcher(rgb8=True): the oracle chain's mosaic bytes and matches, and a device high-water mark at
    least 12 B per input pixel (the f32 copies) below the convert-then-f32 chain's on the same job."""
    from openpano_b200.stitcher import ordered_pairs, unpack_rgb8_mosaic
    monkeypatch.setenv("PANO_CACHE_MB", "0")
    imgs, org = synth.make_stack(5, 1500, 1112, 500, 2)
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    items, geom = synth.translation_blend_setup(org, 1500, 1112)
    p = default_params(ordered_input=1)
    pairs = ordered_pairs(len(pix))
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    new_mark, out, matches = _pipelined_job(pix, pairs, items, geom, p, convert_first=False)
    old_mark, old_out, old_matches = _pipelined_job(pix, pairs, items, geom, p, convert_first=True)
    assert len(matches) == len(old_matches) and all(np.array_equal(a, b) for a, b in zip(matches, old_matches))
    f32 = [orc.read_img_rgb8(a) for a in pix]
    descs = [orc.sift_detect(im, p)[1] for im in f32]
    for (i, j), m in zip(pairs, matches):
        assert np.array_equal(m, orc.match(descs[i], descs[j], p))
    want_rect, want = orc.crop(orc.blend(f32, items, geom, 0, p))
    for buf in (out, old_out):
        rect, px = unpack_rgb8_mosaic(buf, (ow, oh), cropped=True)
        assert np.array_equal(rect, want_rect)
        assert gu.same_bits(px, orc.write_rgb8(want))
    n_px = sum(a.shape[0] * a.shape[1] for a in pix)
    print(f"high-water: convert-then-f32 {old_mark / 2**20:.1f} MB, 8-bit sources {new_mark / 2**20:.1f} MB, "
          f"f32 copies {12 * n_px / 2**20:.1f} MB")
    assert old_mark - new_mark >= 12 * n_px, (old_mark, new_mark, 12 * n_px)


def test_invalid_calls(engine, orc):
    from openpano_b200.capi import LIB
    pix, items, geom = _stack_pix(3)
    n = len(pix)
    d_pix = [engine.dev_alloc(x.nbytes) for x in pix]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    d_out = engine.dev_alloc(tw * th * 12)
    p = default_params()
    vp, ip = C.c_void_p, C.c_int

    def arr(t, vals):
        return (t * max(len(vals), 1))(*vals)

    ws, hs = [x.shape[1] for x in pix], [x.shape[0] for x in pix]
    try:
        for d, x in zip(d_pix, pix):
            engine.dev_upload(d, x)
        fs = C.c_void_p()

        def sift(fn, ptrs=d_pix, w=ws, h=hs, ch=(3, 3, 3), count=n, params=True, out=True):
            return fn(engine._h, count, arr(vp, ptrs) if ptrs is not None else None, arr(ip, w) if w is not None else None,
                      arr(ip, h) if h is not None else None, arr(ip, ch) if ch is not None else None,
                      C.byref(p) if params else None, C.byref(fs) if out else None)
        host_ptrs = [x.ctypes.data for x in pix]
        for fn, ptrs in ((LIB.pano_sift_detect_batch_rgb8_dev, d_pix), (LIB.pano_sift_detect_batch_rgb8, host_ptrs)):
            assert sift(fn, ptrs, count=0) == -2
            assert sift(fn, None) == -2
            assert sift(fn, ptrs, w=None) == -2
            assert sift(fn, ptrs, h=None) == -2
            assert sift(fn, ptrs, ch=None) == -2
            assert sift(fn, ptrs, params=False) == -2
            assert sift(fn, ptrs, out=False) == -2
            assert sift(fn, [ptrs[0], None, ptrs[2]]) == -2
            for bad in (0, 2, 4):
                assert sift(fn, ptrs, ch=(3, bad, 3)) == -2
            assert sift(fn, ptrs, w=[ws[0], 1, ws[2]]) == -2
            assert sift(fn, ptrs, h=[hs[0], hs[1], 1]) == -2
        assert LIB.pano_sift_detect_batch_rgb8_dev(None, n, arr(vp, d_pix), arr(ip, ws), arr(ip, hs), arr(ip, [3] * n),
                                                   C.byref(p), C.byref(fs)) == -2

        blend_args, g = engine._blend_args([None] * n, [x.shape[:2] for x in pix], items, geom)

        def blend(ptrs=d_pix, ch=(3, 3, 3), count=n, imgs=True, geo=True, out=d_out, ow=tw, oh=th):
            return LIB.pano_blend_rgb8_dev(engine._h, count, blend_args if imgs else None,
                                           arr(vp, ptrs) if ptrs is not None else None,
                                           arr(ip, ch) if ch is not None else None, C.byref(g) if geo else None, 0,
                                           C.byref(p), vp(out), ow, oh)
        assert blend(count=0) == -2
        assert blend(ptrs=None) == -2
        assert blend(ch=None) == -2
        assert blend(imgs=False) == -2
        assert blend(geo=False) == -2
        assert blend(out=None) == -2
        assert blend(ptrs=[d_pix[0], None, d_pix[2]]) == -2
        for bad in (0, 2, 4):
            assert blend(ch=(3, 3, bad)) == -2
        assert blend(ow=tw + 1) == -2
        small, sg = engine._blend_args([None] * n, [(1, 240)] + [x.shape[:2] for x in pix[1:]], items, geom)
        assert LIB.pano_blend_rgb8_dev(engine._h, n, small, arr(vp, d_pix), arr(ip, [3] * n), C.byref(sg), 0,
                                       C.byref(p), vp(d_out), tw, th) == -2
    finally:
        for d in d_pix + [d_out]:
            engine.dev_free(d)
    # the context is still usable
    f32 = [orc.read_img_rgb8(x) for x in pix]
    assert _same_features(_features(engine.sift_detect_batch_rgb8(pix)), _features(engine.sift_detect_batch(f32)))
    want, got = _blend_both(engine, pix, items, geom, 0, p)
    assert gu.same_bits(got, want) and gu.same_bits(want, orc.blend(f32, items, geom, 0, p))


def test_cpp_detect_batch_rgb8_equals_reference_read_img(tmp_path):
    """B200SIFTDetector::detect_batch_rgb8 (openpano_b200/host/pano_host.hh) on interleaved bytes next to the reference's
    read_img + SIFTDetector::detect_feature on PPM / PGM files of the same pixels (oracle/_ref/rgb8_sift_test)."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/rgb8_sift_test not built (needs the reference sources at build time)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(tmp_path)], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "RGB8 SIFT TEST OK" in out.stdout
    assert out.stdout.count("identical") == 4
