"""GPU: every blend entry point against the oracle where the inverse map reaches the lens horizon (360° canvases,
wide flat yaw, adversarial inverse maps: tests/wide_geometry.py), linear and multiband, compared as raw uint32 so
that NaN bits count; and write_rgb's f32 -> u8 conversion on values outside [0, 1] through every encoder path.

The reference (and the oracle, pinned to it by tests/test_oracle_wide_geometry.py) converts with x86-64's rule:
a NaN, infinite or >= 2^31 coordinate floors to INT_MIN, so the image is Color::NO there, and a product >= 2^31,
+inf or NaN encodes as 0.  The kernels convert through f2i_x86 (common.cuh) to match."""
import numpy as np
import pytest

from openpano_b200._abi import default_params
from openpano_b200.capi import PIX_FORMATS, SIZE_MAX
from openpano_b200.stitcher import mosaic_rgb8_sweep
from tests import pix_util as xu
from tests import wide_geometry as wg
from tests.test_gpu_blend_strips import _as_format

pytestmark = pytest.mark.gpu
BANDS = [0, 1, 3]
_cache = {}


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = _bits(got) != _bits(want)
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:5].tolist())


def _case(orc, name, bands, rgb8=False, lazy=1, ordered=0):
    """(sources, items, geom, params, the oracle's mosaic); rgb8: 8-bit sources, the oracle on read_img's f32."""
    key = (name, bands, rgb8, lazy, ordered)
    if key not in _cache:
        imgs, items, geom = wg.geometry(name)
        p = default_params(multiband=bands, lazy_read=lazy, ordered_input=ordered)
        srcs = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs] if rgb8 else imgs
        f32 = [orc.read_img_rgb8(x) for x in srcs] if rgb8 else imgs
        want = orc.blend(f32, items, geom, bands, p)
        assert not np.isnan(want).any()
        _cache[key] = (srcs, items, geom, p, want)
    return _cache[key]


def _canvas(items):
    return max(it[2] for it in items), max(it[3] for it in items)


def _upload(engine, arrs):
    ptrs = [engine.dev_alloc(max(a.nbytes, 256)) for a in arrs]
    for d, a in zip(ptrs, arrs):
        engine.dev_upload(d, np.ascontiguousarray(a))
    return ptrs


def _free(engine, ptrs):
    for d in ptrs:
        engine.dev_free(d)


@pytest.mark.parametrize("bands", BANDS)
@pytest.mark.parametrize("name", wg.GEOMETRIES)
def test_blend_f32(engine, orc, name, bands):
    """pano_blend and pano_blend_dev; with bands 0 every (lazy_read, ordered_input)."""
    for lazy, ordered in ((1, 0), (0, 0), (1, 1), (0, 1)) if bands == 0 else ((1, 0),):
        imgs, items, geom, p, want = _case(orc, name, bands, lazy=lazy, ordered=ordered)
        _same(engine.blend(imgs, items, geom, bands, p), want, ("blend", lazy, ordered))
    ow, oh = _canvas(items)
    d_imgs = _upload(engine, imgs)
    d_out = engine.dev_alloc(ow * oh * 12)
    try:
        engine.blend_dev(d_imgs, [im.shape[:2] for im in imgs], items, geom, d_out, ow, oh, bands, p)
        got = np.empty((oh, ow, 3), np.float32)
        engine.dev_download(got, d_out)
    finally:
        _free(engine, d_imgs + [d_out])
    _same(got, want, "blend_dev")


@pytest.mark.parametrize("bands", BANDS)
@pytest.mark.parametrize("name", wg.GEOMETRIES)
def test_blend_rgb8_layouts(engine, orc, name, bands):
    """pano_blend_rgb8_dev from interleaved RGB, lodepng's RGBA and CImg's planar sources."""
    pix, items, geom, p, want = _case(orc, name, bands, rgb8=True)
    shapes = [x.shape[:2] for x in pix]
    ow, oh = _canvas(items)
    for fmt in ("rgb", "rgba", "planar"):
        srcs = [_as_format(x, fmt) for x in pix]
        d_pix = _upload(engine, srcs)
        d_out = engine.dev_alloc(ow * oh * 12)
        try:
            engine.blend_rgb8_dev(d_pix, [PIX_FORMATS[fmt]] * len(srcs), shapes, items, geom, d_out, ow, oh, bands, p)
            got = np.empty((oh, ow, 3), np.float32)
            engine.dev_download(got, d_out)
        finally:
            _free(engine, d_pix + [d_out])
        _same(got, want, fmt)


@pytest.mark.parametrize("bands", BANDS)
@pytest.mark.parametrize("name", wg.GEOMETRIES)
def test_blend_row_strips(engine, orc, name, bands):
    """pano_blend_rows_dev (f32) and pano_blend_rows_rgb8_dev on uneven row strips, concatenated."""
    for rgb8 in (False, True):
        srcs, items, geom, p, want = _case(orc, name, bands, rgb8=rgb8)
        ow, oh = _canvas(items)
        cuts = sorted({0, 1, 7, oh // 3, oh // 3 + 1, oh - 2, oh})
        d_src = _upload(engine, srcs)
        d_out = engine.dev_alloc(ow * oh * 12)
        parts = []
        try:
            for r0, r1 in zip(cuts[:-1], cuts[1:]):
                if rgb8:
                    engine.blend_rows_rgb8_dev(d_src, [3] * len(srcs), [x.shape[:2] for x in srcs], items, geom, d_out,
                                               ow, oh, r0, r1, bands, p)
                else:
                    engine.blend_rows_dev(d_src, [x.shape[:2] for x in srcs], items, geom, d_out, ow, oh, r0, r1, bands,
                                          p)
                part = np.empty((r1 - r0, ow, 3), np.float32)
                engine.dev_download(part, d_out)
                parts.append(part)
        finally:
            _free(engine, d_src + [d_out])
        _same(np.concatenate(parts), want, ("rows", rgb8))


@pytest.mark.parametrize("bands", BANDS)
@pytest.mark.parametrize("name", wg.GEOMETRIES)
def test_blend_lazy_windows(engine, orc, name, bands):
    """A blend stream fed in windows of 1, 2 and the rest: f32 sources, and 8-bit ones in one layout per window."""
    imgs, items, geom, p, want = _case(orc, name, bands)
    _same(engine.blend_lazy(imgs, items, geom, bands, p, window=[1, 2, len(imgs)]), want, "f32")
    pix, items, geom, p, want = _case(orc, name, bands, rgb8=True)
    fmts = ["rgba", "planar", "rgb"]
    srcs = []
    for q, (k0, n) in enumerate(((0, 1), (1, 2), (3, len(pix)))):
        srcs += [_as_format(x, fmts[q]) for x in pix[k0:k0 + n]]
    _same(engine.blend_lazy(srcs, items, geom, bands, p, window=[1, 2, len(pix)], fmt=fmts), want, "rgb8")


@pytest.mark.parametrize("bands", BANDS)
@pytest.mark.parametrize("name", wg.GEOMETRIES)
def test_blend_sweep(engine, orc, name, bands):
    """The blend sweep's 8-bit mosaic, crop on and off, against crop + write_rgb of the oracle's mosaic."""
    pix, items, geom, p, want = _case(orc, name, bands, rgb8=True)
    rect, cropped = orc.crop(want)
    for crop, out in ((True, "rgb"), (False, "rgba"), (True, "planar")):
        rgb = orc.write_rgb8(cropped if crop else want)
        ref = {"rgb": rgb, "rgba": xu.to_rgba(rgb), "planar": xu.to_planar(rgb)}[out]
        got_rect, got = mosaic_rgb8_sweep(engine, items, geom, bands, pix, 37, SIZE_MAX, out, crop, params=p)
        if crop:
            assert np.array_equal(got_rect, rect), (got_rect, rect)
        assert np.array_equal(got, ref), (crop, out)


# ----------------------------------------------------------------------------------------------- f32 -> u8
def _u8_mosaics():
    """The sweep mosaic, and its absolute values inside a Color::NO frame (so that crop keeps all of them)."""
    m = wg.u8_sweep_mosaic()
    framed = np.full((m.shape[0] + 4, m.shape[1] + 6, 3), -1.0, np.float32)
    framed[2:-2, 3:-3] = np.abs(m)
    return [m, framed]


def test_u8_sweep_conversions(engine, orc):
    """pano_mat32f_to_rgb8_dev and pano_mat32f_to_pix8_dev (through crop_write_rgb8 / crop_write_pix8), crop on and
    off, every layout: the bytes of write_rgb on x86-64."""
    for m in _u8_mosaics():
        want = wg.x86_write_rgb(m)
        assert np.array_equal(orc.write_rgb8(m), want)
        _, got = engine.crop_write_rgb8(m, crop=False)
        assert np.array_equal(got, want), np.argwhere(got != want)[:5].tolist()
        rect, cropped = orc.crop(m)
        cw = wg.x86_write_rgb(cropped)
        got_rect, got = engine.crop_write_rgb8(m, crop=True)
        assert np.array_equal(got_rect, rect) and np.array_equal(got, cw)
        for fmt, conv in (("rgba", xu.to_rgba), ("planar", xu.to_planar)):
            _, got = engine.crop_write_pix8(m, crop=False, fmt=fmt)
            assert np.array_equal(got, conv(want)), fmt
            got_rect, got = engine.crop_write_pix8(m, crop=True, fmt=fmt)
            assert np.array_equal(got_rect, rect) and np.array_equal(got, conv(cw)), fmt


def test_u8_sweep_strip_encoder(engine):
    """The strip writers' path: pano_mat32f_to_rgb8_dev on row strips of the uncropped mosaic, then
    pano_rgb8_crop_to_pix8_dev in every layout."""
    m = _u8_mosaics()[1]
    h, w = m.shape[:2]
    want = wg.x86_write_rgb(m)
    d_mat, d_rgb, d_out = _upload(engine, [m])[0], engine.dev_alloc(h * w * 3), engine.dev_alloc(h * w * 4)
    try:
        for r0 in range(0, h, 5):
            r1 = min(h, r0 + 5)
            engine.mat32f_to_rgb8_dev(d_mat + r0 * w * 12, w, r1 - r0, 0, d_rgb + r0 * w * 3)
        for fmt, shape, conv in (("rgb", (h, w, 3), lambda x: x), ("rgba", (h, w, 4), xu.to_rgba),
                                 ("planar", (3, h, w), xu.to_planar)):
            engine.rgb8_crop_to_pix8_dev(d_rgb, w, h, 0, fmt, d_out)
            got = np.empty(shape, np.uint8)
            engine.dev_download(got, d_out)
            assert np.array_equal(got, conv(want)), fmt
    finally:
        _free(engine, [d_mat, d_rgb, d_out])
