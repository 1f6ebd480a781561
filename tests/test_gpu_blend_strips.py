"""GPU: the mosaic strip by strip in bounded device memory.  Row-strip blend streams
(pano_blend_stream_create_rows) concatenated must have the raw bits of pano_blend for every strip partition,
window partition, source kind and pixel format, linear and multiband; pano_blend_stream_needs must follow
pano_blend_rows_rgb8_dev's rule; the crop scan (pano_crop_scan_*) must give pano_crop_rect_dev's rectangle for
every strip partition and orc_crop's past 40,000 columns; and the 8-bit mosaic built from strips must be the
bytes of pano_mat32f_to_pix8_dev on the whole f32 mosaic with its crop rectangle."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests import golden_util as gu
from tests.test_gpu_imgio import _mosaic
from tests.test_gpu_match_warp_blend import _perspective_items

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "blend_strips_test"
MB = 1 << 20
# summed blur half-widths of the multiband levels at GAUSS_WINDOW_FACTOR 6 (include/pano_b200.h)
HALO = {0: 0, 1: 0, 2: 6, 3: 12, 5: 27}


def _pix(imgs):
    return [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]


def _gap_stack():
    """Two rows of images 100 rows apart: canvas rows no image (and no multiband halo) reaches."""
    imgs, org = synth.make_stack(6, 200, 100, 80, 5, rows=2, step_y=200)
    items, geom = synth.translation_blend_setup(org, 200, 100)
    return imgs, items, geom


def _stack(n=7):
    imgs, org = synth.make_stack(n, 240, 180, 70, 23, rows=2, step_y=60)
    items, geom = synth.translation_blend_setup(org, 240, 180)
    return imgs, items, geom


def _canvas(items):
    return max(it[2] for it in items), max(it[3] for it in items)


def _need_rule(items, bands, r0, r1, oh):
    if r0 == 0 and r1 == oh:
        return np.ones(len(items), bool)
    if bands == 0:
        return np.array([y0 < r1 and y1 >= r0 for _, y0, _, y1, _ in items])
    c0 = max(0, r0 - HALO[bands]) if r0 > 0 else -(1 << 40)
    c1 = r1 + HALO[bands] - 1 if r1 < oh else 1 << 40
    return np.array([max(y0, c0) <= min(y1, c1) for _, y0, _, y1, _ in items])


def _windows(n, window):
    window = window or n
    return [(k, min(n, k + window)) for k in range(0, n, window)]


def _strips(engine, srcs, shapes, items, geom, bands, p, heights, window, kind=None, channels=3, fmt=None):
    """Concatenated row-strip streams; every image a strip does not need is passed as None."""
    ow, oh = _canvas(items)
    assert sum(heights) == oh
    out, r0 = [], 0
    for hgt in heights:
        r1 = r0 + hgt
        s = engine.blend_stream_rows(shapes, items, geom, r0, r1, bands, p)
        try:
            need = s.needs()
            assert np.array_equal(need, _need_rule(items, bands, r0, r1, oh)), (r0, r1)
            for k0, k1 in _windows(len(items), window):
                s.add([srcs[k] if need[k] else None for k in range(k0, k1)], kind, channels, fmt)
            out.append(s.finish())
        finally:
            s.close()
        r0 = r1
    return np.concatenate(out)


def _heights(name, oh, bands):
    H = HALO[bands]
    seq = {"1": [1], "7": [7], "H": [max(H, 2)], "H+1": [H + 1], "uneven": [5, 40, 3, 61, 17], "whole": [oh]}[name]
    out, k = [], 0
    while sum(out) < oh:
        out.append(min(seq[k % len(seq)], oh - sum(out)))
        k += 1
    return out


@pytest.mark.parametrize("bands", [0, 1, 2, 5])
@pytest.mark.parametrize("part", ["1", "7", "H", "H+1", "uneven", "whole"])
def test_strip_partitions_bit_exact(engine, bands, part):
    imgs, items, geom = _gap_stack()
    pix = _pix(imgs)
    f32 = [engine.read_img_rgb8(x) for x in pix]
    want = engine.blend(f32, items, geom, bands)
    assert (want[..., 0] == -1).all(axis=1).sum() > 60          # empty canvas rows
    heights = _heights(part, want.shape[0], bands)
    got = _strips(engine, pix, [x.shape[:2] for x in pix], items, geom, bands, None, heights, 3)
    assert gu.same_bits(got, want)


@pytest.mark.parametrize("bands", [0, 5])
def test_strip_no_image_reaches_is_all_minus_one(engine, bands):
    imgs, items, geom = _gap_stack()
    ow, oh = _canvas(items)
    s = engine.blend_stream_rows([im.shape[:2] for im in imgs], items, geom, 145, 155, bands)
    try:
        assert not s.needs().any()
        s.add([None] * 2)
        s.add([None] * 4)
        got = s.finish()
    finally:
        s.close()
    assert got.shape == (10, ow, 3) and (got == -1).all()


@pytest.mark.parametrize("lazy,ordered", [(1, 0), (1, 1), (0, 0), (0, 1)])
@pytest.mark.parametrize("window", [1, 3, None])
def test_linear_settings_and_windows(engine, orc, lazy, ordered, window):
    imgs, items, geom = _stack(7)
    pix = _pix(imgs)
    p = default_params(lazy_read=lazy, ordered_input=ordered)
    f32 = [orc.read_img_rgb8(x) for x in pix]
    want = engine.blend(f32, items, geom, 0, p)
    if window is None:
        assert gu.same_bits(want, orc.blend(f32, items, geom, 0, p))
    got = _strips(engine, pix, [x.shape[:2] for x in pix], items, geom, 0, p, _heights("uneven", want.shape[0], 0), window)
    assert gu.same_bits(got, want)


@pytest.mark.parametrize("window", [1, 3, None])
@pytest.mark.parametrize("bands", [2, 5])
def test_multiband_windows(engine, orc, bands, window):
    imgs, items, geom = _stack(7)
    pix = _pix(imgs)
    f32 = [engine.read_img_rgb8(x) for x in pix]
    want = engine.blend(f32, items, geom, bands)
    if window is None and bands == 5:
        assert gu.same_bits(want, orc.blend([orc.read_img_rgb8(x) for x in pix], items, geom, bands))
    got = _strips(engine, pix, [x.shape[:2] for x in pix], items, geom, bands, None,
                  _heights("H+1", want.shape[0], bands), window)
    assert gu.same_bits(got, want)


@pytest.mark.parametrize("projection", [0, 1, 2])
@pytest.mark.parametrize("bands", [0, 3])
def test_strip_projections_bit_exact(engine, projection, bands):
    imgs, org = synth.make_stack(4, 300, 200, 100, 7)
    items, geom = _perspective_items(org, 4, projection)
    pix = _pix(imgs)
    f32 = [engine.read_img_rgb8(x) for x in pix]
    want = engine.blend(f32, items, geom, bands)
    assert (want < 0).mean() < 0.9
    for part in ("7", "uneven"):
        got = _strips(engine, pix, [x.shape[:2] for x in pix], items, geom, bands, None,
                      _heights(part, want.shape[0], bands), 1)
        assert gu.same_bits(got, want), part


def _as_format(x, fmt):
    if fmt == "grey":
        return np.ascontiguousarray(x[..., 1])
    if fmt == "rgba":
        a = np.random.RandomState(int(x[0, 0, 0])).randint(0, 256, x.shape[:2] + (1,)).astype(np.uint8)
        return np.ascontiguousarray(np.concatenate([x, a], axis=2))
    if fmt == "planar":
        return np.ascontiguousarray(x.transpose(2, 0, 1))
    return x


@pytest.mark.parametrize("fmt", ["grey", "rgb", "rgba", "planar"])
@pytest.mark.parametrize("bands", [0, 2])
def test_source_kinds_and_formats(engine, fmt, bands):
    """Device and host sources, f32 and 8-bit in every PANO_PIX_* format, pinned and pageable; NULL for the
    images a strip does not need."""
    from openpano_b200.capi import (PIX_FORMATS, SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_DEV, SRC_RGB8_HOST, Engine)
    imgs, items, geom = _gap_stack()
    pix = [_as_format(x, fmt) for x in _pix(imgs)]
    code = PIX_FORMATS[fmt]
    f32 = [engine.read_img_rgb8(x, fmt=fmt) for x in pix]
    shapes = [x.shape[:2] for x in f32]
    want = engine.blend(f32, items, geom, bands)
    heights = _heights("uneven", want.shape[0], bands)
    d_f32 = [engine.dev_alloc(x.nbytes) for x in f32]
    d_pix = [engine.dev_alloc(x.nbytes) for x in pix]
    h_f32 = [Engine.host_alloc(x.nbytes) for x in f32]
    h_pix = [Engine.host_alloc(x.nbytes) for x in pix]
    try:
        for d, h, x in zip(d_f32 + d_pix, h_f32 + h_pix, f32 + pix):
            engine.dev_upload(d, x)
            C.memmove(h, x.ctypes.data, x.nbytes)
        for kind, ptrs, ch in ((SRC_F32_DEV, d_f32, 3), (SRC_F32_HOST, h_f32, 3), (SRC_RGB8_DEV, d_pix, code),
                               (SRC_RGB8_HOST, h_pix, code)):
            got = _strips(engine, ptrs, shapes, items, geom, bands, None, heights, 2, kind, ch)
            assert gu.same_bits(got, want), kind
        assert gu.same_bits(_strips(engine, pix, shapes, items, geom, bands, None, heights, 3, fmt=fmt), want)
        assert gu.same_bits(_strips(engine, f32, shapes, items, geom, bands, None, heights, None), want)
    finally:
        for d in d_f32 + d_pix:
            engine.dev_free(d)
        for h in h_f32 + h_pix:
            Engine.host_free(h)


def test_misuse_is_invalid_and_sticky(engine):
    from openpano_b200.capi import LIB, PanoError, SRC_RGB8_HOST
    imgs, items, geom = _gap_stack()
    pix = _pix(imgs)
    shapes = [x.shape[:2] for x in pix]
    arr, g = engine._blend_args([None] * 6, shapes, items, geom)
    p = default_params()
    ow, oh = _canvas(items)
    out = np.empty((oh, ow, 3), np.float32)
    fp = C.POINTER(C.c_float)
    h = C.c_void_p()
    for r0, r1 in ((-1, 10), (0, oh + 1), (20, 20), (30, 10)):
        assert LIB.pano_blend_stream_create_rows(engine._h, 6, arr, C.byref(g), 0, C.byref(p), ow, oh, r0, r1,
                                                 C.byref(h)) == -2, (r0, r1)
    assert LIB.pano_blend_stream_create_rows(engine._h, 6, arr, C.byref(g), 0, C.byref(p), ow + 1, oh, 0, 10,
                                             C.byref(h)) == -2
    assert LIB.pano_blend_stream_needs(None, None) == -2
    for bands in (0, 3):
        assert LIB.pano_blend_stream_create_rows(engine._h, 6, arr, C.byref(g), bands, C.byref(p), ow, oh, 0, 40,
                                                 C.byref(h)) == 0
        try:
            assert LIB.pano_blend_stream_needs(h, None) == -2
            flags = np.zeros(6, np.uint8)
            assert LIB.pano_blend_stream_needs(h, flags.ctypes.data) == 0
            assert flags[0] == 1 and flags[3] == 0
            srcs = (C.c_void_p * 6)(*[None] * 6)           # image 0 is needed: NULL is a misuse
            assert LIB.pano_blend_stream_add(h, 0, 6, srcs, SRC_RGB8_HOST, 3) == -2
            srcs = (C.c_void_p * 6)(*[x.ctypes.data for x in pix])
            assert LIB.pano_blend_stream_add(h, 0, 6, srcs, SRC_RGB8_HOST, 3) == -2, "not sticky"
            assert LIB.pano_blend_stream_finish(h, out.ctypes.data_as(fp)) == -2, "not sticky"
        finally:
            LIB.pano_blend_stream_free(h)
    s = engine.blend_stream_rows(shapes, items, geom, 0, 40)
    try:
        with pytest.raises(PanoError) as ei:
            s.add([None, pix[1]])
        assert ei.value.code == -2
        with pytest.raises(PanoError):
            s.add(pix[2:])
    finally:
        s.close()
    # the context is still usable
    f32 = [engine.read_img_rgb8(x) for x in pix]
    assert gu.same_bits(_strips(engine, pix, shapes, items, geom, 0, None, [40, oh - 40], 6),
                        engine.blend(f32, items, geom, 0))


# ------------------------------------------------------------------ crop scan
def _scan_rect(engine, m, heights):
    h, w = m.shape[:2]
    d = engine.dev_alloc(m.nbytes)
    scan = engine.crop_scan(w, h)
    try:
        engine.dev_upload(d, m)
        r0 = 0
        for hgt in heights:
            scan.add_dev(d + r0 * w * 12, hgt)
            r0 += hgt
        return scan.rect()
    finally:
        scan.close()
        engine.dev_free(d)


def _crop_rect_dev(engine, m):
    h, w = m.shape[:2]
    d, d_rect = engine.dev_alloc(m.nbytes), engine.dev_alloc(256)
    rect = np.zeros(4, np.int32)
    try:
        engine.dev_upload(d, m)
        engine.crop_rect_dev(d, w, h, d_rect)
        engine.dev_download(rect, d_rect)
    finally:
        engine.dev_free(d)
        engine.dev_free(d_rect)
    return rect


def _partitions(h):
    rng = np.random.RandomState(h)
    parts = [[h], [1] * h, [32] * (h // 32) + ([h % 32] if h % 32 else []), [7] * (h // 7) + ([h % 7] if h % 7 else [])]
    cuts = sorted(set(rng.randint(1, h, size=min(h - 1, 5)).tolist())) if h > 1 else []
    parts.append([b - a for a, b in zip([0] + cuts, cuts + [h])])
    return parts


@pytest.mark.parametrize("h,w,holes,border", [
    (40, 60, 4, False), (97, 2500, 3, True), (200, 1024, 30, True), (70, 300, 0, True), (12, 6000, -1, False)])
def test_crop_scan_equals_crop_rect(engine, h, w, holes, border):
    rng = np.random.RandomState(h + w)
    m = _mosaic(rng, h, w, max(holes, 0), border)
    if holes < 0:      # per-column noise: thousands of height runs per line (per-column search path)
        for k in range(w):
            m[:rng.randint(0, 6), k] = -1
    want = _crop_rect_dev(engine, m)
    assert want[2] * want[3] > 0
    for heights in _partitions(h):
        assert np.array_equal(_scan_rect(engine, m, heights), want), heights


def test_crop_scan_degenerate(engine, orc):
    cases = {
        "all NO": -np.ones((40, 7, 3), np.float32),
        "one row": np.random.RandomState(1).rand(1, 50, 3).astype(np.float32),
        "one column": np.random.RandomState(2).rand(45, 1, 3).astype(np.float32),
    }
    ties = np.zeros((40, 20, 3), np.float32)           # two equal-area rectangles: the first in (line, column) order
    ties[:, 9:11] = -1
    cases["ties"] = ties
    stacked = np.zeros((64, 30, 3), np.float32)        # equal areas in different strips: the upper one wins
    stacked[30:34] = -1
    cases["ties across strips"] = stacked
    hole_row = np.random.RandomState(3).rand(50, 40, 3).astype(np.float32)
    hole_row[::9, 5] = -1
    hole_row[1, :] = -1
    cases["holes"] = hole_row
    for name, m in cases.items():
        want = orc.crop(m)[0]
        assert np.array_equal(_crop_rect_dev(engine, m), want), name
        for heights in _partitions(m.shape[0]):
            assert np.array_equal(_scan_rect(engine, m, heights), want), (name, heights)


@pytest.mark.parametrize("w", [40001, 57313, 80000])
def test_crop_scan_wide_equals_oracle(engine, orc, w):
    rng = np.random.RandomState(w)
    h = 48
    m = np.zeros((h, w, 3), np.float32)
    yy, xx = np.mgrid[0:h, 0:w]
    m[(yy < 2 + 6.0 * xx / w) | (yy > h - 3 - 9.0 * (w - xx) / w)] = -1
    for _ in range(40):
        y0, x0 = rng.randint(0, h), rng.randint(0, w)
        m[y0:y0 + rng.randint(1, 4), x0:x0 + rng.randint(1, 3000)] = -1
    for k in rng.randint(0, w, 2000):                # per-column noise at the top: the fallback search path
        m[:rng.randint(0, 5), k] = -1
    want = orc.crop(m)[0]
    assert want[2] * want[3] > 100000
    for heights in ([h], [5, 11, 32], [1] * h):
        assert np.array_equal(_scan_rect(engine, m, heights), want), heights
    from openpano_b200.capi import PanoError
    with pytest.raises(PanoError):
        engine.crop_scan(80001, h)


def test_crop_scan_misuse(engine):
    from openpano_b200.capi import LIB, PanoError
    h = C.c_void_p()
    assert LIB.pano_crop_scan_create(engine._h, 0, 5, C.byref(h)) == -2
    assert LIB.pano_crop_scan_create(engine._h, 5, 0, C.byref(h)) == -2
    assert LIB.pano_crop_scan_create(None, 5, 5, C.byref(h)) == -2
    assert LIB.pano_crop_scan_add_dev(None, None, 1) == -2
    m = np.zeros((10, 8, 3), np.float32)
    d = engine.dev_alloc(m.nbytes)
    try:
        engine.dev_upload(d, m)
        for name, steps in {"too many lines": [(d, 6), (d, 5)], "null strip": [(0, 3)], "no lines": [(d, 0)],
                            "rect early": [(d, 4), None]}.items():
            scan = engine.crop_scan(8, 10)
            try:
                with pytest.raises(PanoError) as ei:
                    for st in steps:
                        scan.rect() if st is None else scan.add_dev(*st)
                assert ei.value.code == -2, name
                with pytest.raises(PanoError):     # sticky
                    scan.add_dev(d, 1)
                with pytest.raises(PanoError):
                    scan.rect()
            finally:
                scan.close()
        assert np.array_equal(_scan_rect(engine, m, [3, 7]), [0, 0, 8, 10])
    finally:
        engine.dev_free(d)
    LIB.pano_crop_scan_free(None)


# ------------------------------------------------------------------ 8-bit output
@pytest.mark.parametrize("fmt", ["rgb", "rgba", "planar"])
def test_rgb8_crop_equals_f32_conversion(engine, fmt):
    from openpano_b200.capi import PIX_FORMATS
    rng = np.random.RandomState(9)
    h, w = 77, 301
    m = _mosaic(rng, h, w, 12, True)
    bpp = 4 if fmt == "rgba" else 3
    d_m, d_rgb, d_rect = engine.dev_alloc(m.nbytes), engine.dev_alloc(h * w * 3), engine.dev_alloc(256)
    d_a, d_b = engine.dev_alloc(h * w * bpp), engine.dev_alloc(h * w * bpp)
    try:
        engine.dev_upload(d_m, m)
        engine.crop_rect_dev(d_m, w, h, d_rect)
        engine.mat32f_to_rgb8_dev(d_m, w, h, 0, d_rgb)
        for rect in (d_rect, 0):
            engine.mat32f_to_pix8_dev(d_m, w, h, rect, fmt, d_a)
            engine.rgb8_crop_to_pix8_dev(d_rgb, w, h, rect, PIX_FORMATS[fmt], d_b)
            a, b = np.empty(h * w * bpp, np.uint8), np.empty(h * w * bpp, np.uint8)
            engine.dev_download(a, d_a)
            engine.dev_download(b, d_b)
            r = np.zeros(4, np.int32)
            engine.dev_download(r, d_rect)
            nb = (int(r[2]) * int(r[3]) if rect else h * w) * bpp
            assert 0 < nb < h * w * bpp or not rect
            assert gu.same_bits(a[:nb], b[:nb]), (fmt, rect)
    finally:
        for d in (d_m, d_rgb, d_rect, d_a, d_b):
            engine.dev_free(d)


@pytest.mark.parametrize("bands", [0, 5])
@pytest.mark.parametrize("fmt", ["rgb", "rgba", "planar"])
def test_mosaic_rgb8_strips_equals_whole_canvas(engine, bands, fmt):
    from openpano_b200.stitcher import mosaic_rgb8_strips
    imgs, items, geom = _stack(7)
    items = items[:3] + items[4:]                     # a hole, so that crop has work to do
    imgs = imgs[:3] + imgs[4:]
    pix = _pix(imgs)
    f32 = [engine.read_img_rgb8(x) for x in pix]
    mos = engine.blend(f32, items, geom, bands)
    for crop in (True, False):
        want_rect, want = engine.crop_write_pix8(mos, crop, fmt)
        for strip_rows, window in ((37, 1), (1000, None), (64, 3)):
            rect, got = mosaic_rgb8_strips(engine, items, geom, bands, pix, strip_rows, window, fmt, crop)
            assert (rect is None) == (not crop)
            if crop:
                assert np.array_equal(rect, want_rect)
                assert want_rect[2] * want_rect[3] < mos.shape[0] * mos.shape[1]
            assert gu.same_bits(got, want), (crop, strip_rows, window)


@pytest.mark.parametrize("kind", ["rgb8_dev", "rgb8_host_pinned", "f32_dev"])
def test_mosaic_rgb8_strips_from_pointers(engine, kind):
    """mosaic_rgb8_strips from raw pointers (kind / channels / shapes): device and pinned host sources."""
    from openpano_b200.capi import PIX_RGBA, SRC_F32_DEV, SRC_RGB8_DEV, SRC_RGB8_HOST, Engine
    from openpano_b200.stitcher import mosaic_rgb8_strips
    imgs, items, geom = _gap_stack()
    pix = [_as_format(x, "rgba") for x in _pix(imgs)]
    f32 = [engine.read_img_rgb8(x, fmt="rgba") for x in pix]
    shapes = [x.shape[:2] for x in f32]
    want_rect, want = engine.crop_write_pix8(engine.blend(f32, items, geom, 2), True, "planar")
    src = f32 if kind == "f32_dev" else pix
    host = kind == "rgb8_host_pinned"
    ptrs = [Engine.host_alloc(x.nbytes) if host else engine.dev_alloc(x.nbytes) for x in src]
    try:
        for q, x in zip(ptrs, src):
            if host:
                C.memmove(q, x.ctypes.data, x.nbytes)
            else:
                engine.dev_upload(q, x)
        code, ch = {"rgb8_dev": (SRC_RGB8_DEV, PIX_RGBA), "rgb8_host_pinned": (SRC_RGB8_HOST, PIX_RGBA),
                    "f32_dev": (SRC_F32_DEV, 3)}[kind]
        rect, got = mosaic_rgb8_strips(engine, items, geom, 2, ptrs, 41, 2, "planar", kind=code, channels=ch,
                                       shapes=shapes)
    finally:
        for q in ptrs:
            Engine.host_free(q) if host else engine.dev_free(q)
    assert np.array_equal(rect, want_rect)
    assert gu.same_bits(got, want)


def test_cpp_write_strips_equals_reference(tmp_path):
    """B200PixelBlender::write_strips (openpano_b200/host/pano_host_io.hh) next to the reference's blenders, crop() and
    write_rgb() on PNG and PPM files, strip heights 1 to a whole canvas, and a canvas over 40,000 columns
    (oracle/_ref/blend_strips_test)."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/blend_strips_test not built (needs the reference sources at build time)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(tmp_path)], capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "BLEND STRIPS TEST OK" in out.stdout
    assert out.stdout.count("identical") == 16 + 2 + 16 + 2


def test_wide_canvas_end_to_end_against_oracle(engine, orc):
    """A canvas over 40,000 columns: blend, crop and write_rgb on the oracle against the strips, byte for byte."""
    from openpano_b200.stitcher import mosaic_rgb8_strips
    n, w, h = 40, 1200, 90
    imgs, org = synth.make_stack(n, w, h, 1000, 61)
    org = [(x, y + (k * 7) % 23) for k, (x, y) in enumerate(org)]
    items, geom = synth.translation_blend_setup(org, w, h)
    ow, oh = _canvas(items)
    assert ow > 40000
    pix = _pix(imgs)
    f32 = [orc.read_img_rgb8(x) for x in pix]
    mos = orc.blend(f32, items, geom, 0)
    want_rect, want = orc.crop(mos)
    assert 0 < want_rect[3] < oh
    rect, got = mosaic_rgb8_strips(engine, items, geom, 0, pix, 32, 4)
    assert np.array_equal(rect, want_rect)
    assert gu.same_bits(got, orc.write_rgb8(want))


# ------------------------------------------------------------------ memory
def _strip_state(items, tw, r0, r1, th, bands):
    """A strip stream's canvas state as include/pano_b200.h states it (finish()'s output included)."""
    if bands == 0:
        return 16 * tw * (r1 - r0)
    c0 = max(0, r0 - HALO[bands]) if r0 > 0 else 0
    c1 = r1 + HALO[bands] - 1 if r1 < th else th
    roi = 0
    for x0, y0, x1, y1, _ in items:
        y0, y1 = max(y0, c0), min(y1, c1)
        if y0 <= y1:
            roi += -(-(x1 - x0 + 1) // 32) * 32 * (y1 - y0 + 1)
    return 33 * roi + tw * (r1 - r0) + 12 * tw * (r1 - r0)


@pytest.mark.parametrize("bands", [0, 5])
def test_memory_bound(monkeypatch, bands):
    """Strips of 512 rows of a 40-image mosaic: each strip's pool high-water mark stays within its canvas state plus
    two windows of sources plus 64 MB, well below the whole-canvas stream's, and the strips give its bits."""
    from openpano_b200.capi import Engine
    monkeypatch.setenv("PANO_CACHE_MB", "0")
    w, h, n = 2000, 1500, 40
    base = np.random.RandomState(4).randint(0, 256, (h + 4 * 750, w + 7 * 1000, 3), dtype=np.uint8)
    org = [(c * 1000, r * 750) for r in range(5) for c in range(8)]
    pix = [np.ascontiguousarray(base[y:y + h, x:x + w]) for x, y in org]
    items, geom = synth.translation_blend_setup(org, w, h)
    shapes = [x.shape[:2] for x in pix]
    tw, th = _canvas(items)
    eng = Engine(0)
    try:
        eng.trim()
        eng.sync()
        eng.mem_high_water(reset=True)
        s = eng.blend_stream(shapes, items, geom, bands)
        try:
            for k in range(0, n, 2):
                s.add(pix[k:k + 2])
            want = s.finish()
        finally:
            s.close()
        eng.sync()
        whole_mark = eng.mem_high_water(reset=True)
        strips, worst = [], 0
        for r0 in range(0, th, 512):
            r1 = min(th, r0 + 512)
            eng.sync()
            eng.mem_high_water(reset=True)
            s = eng.blend_stream_rows(shapes, items, geom, r0, r1, bands)
            try:
                need = s.needs()
                for k0, k1 in _windows(n, 2):
                    s.add([pix[k] if need[k] else None for k in range(k0, k1)])
                strips.append(s.finish())
            finally:
                s.close()
            eng.sync()
            mark = eng.mem_high_water()
            bound = _strip_state(items, tw, r0, r1, th, bands) + 2 * 2 * pix[0].nbytes + 64 * MB
            assert mark <= bound, (r0, mark / MB, bound / MB)
            worst = max(worst, mark)
        assert gu.same_bits(np.concatenate(strips), want)
        assert worst * 3 < whole_mark, (worst / MB, whole_mark / MB)
        print(f"bands={bands}: strips of 512 rows {worst / MB:.0f} MB at most, whole canvas {whole_mark / MB:.0f} MB")
    finally:
        eng.close()
