"""GPU: the little-planet view straight from a decoded 8-bit image (pano_planet_pix8 / pano_planet_pix8_dev), for
every PANO_PIX_* format.  Every result must have the raw bits of pano_planet on read_img's f32 image of the same
pixels (pano_rgb8_to_mat32f_dev's image) and of the plain-C restatement (tests/planet_util.py) on that image.  Also
the 8-bit chain to write_rgb's encoder buffers, the strip pipeline's cropped mosaic as input, the misuse rules, the
profile names and the C++ drop-in's `planet` command next to the reference's, file bytes."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200.capi import LIB, PIX_GREY, PIX_RGB, PIX_RGB_PLANAR, PIX_RGBA, PanoError
from tests import golden_util as gu
from tests import pix_util as xu
from tests import planet_util as pu

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "planet_pix_test"
OUT_BYTES = pu.SIZE * pu.SIZE * 12
CODE = {"grey": PIX_GREY, "rgb": PIX_RGB, "rgba": PIX_RGBA, "planar": PIX_RGB_PLANAR}
FORMATS = list(CODE)
# (w, h): the reference's CMU1 mosaic, a wide cropped mosaic, a one-row and a one-column strip (no colour, as in
# the reference) and the smallest image with colour
SHAPES = [(8000, 1449), (3000, 600), (700, 1), (1, 450), (2, 2)]
BAD_FORMATS = [0, 2, 4, 5, 0x103, 0x204]


def _buf(w, h, fmt, seed):
    """Random pixels in layout fmt (RGBA with a random fourth byte, which read_img ignores)."""
    rgb = np.random.RandomState(seed).randint(0, 256, size=(h, w, 3)).astype(np.uint8)
    if fmt == "rgba":
        return xu.to_rgba(rgb, alpha_seed=seed + 1)
    if fmt == "planar":
        return xu.to_planar(rgb)
    if fmt == "grey":
        return np.ascontiguousarray(rgb[..., 0])
    return rgb


def _planet_dev(engine, buf, fmt, w, h):
    """planet_pix8_dev on a device copy of buf, into a buffer that starts as NaN (every float must be written)."""
    d_pix, d_out = engine.dev_alloc(max(buf.nbytes, 256)), engine.dev_alloc(OUT_BYTES)
    got = np.empty((pu.SIZE, pu.SIZE, 3), np.float32)
    try:
        engine.dev_upload(d_pix, buf)
        engine.dev_upload(d_out, np.full((pu.SIZE, pu.SIZE, 3), np.nan, np.float32))
        engine.planet_pix8_dev(d_pix, fmt, w, h, d_out)
        engine.dev_download(got, d_out)
    finally:
        engine.dev_free(d_pix)
        engine.dev_free(d_out)
    return got


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{w}x{h}" for w, h in SHAPES])
def test_planet_pix8_bit_exact(engine, shape, fmt):
    w, h = shape
    buf = _buf(w, h, fmt, seed=w + 7 * h + len(fmt))
    f32 = engine.read_img_rgb8(buf, fmt)                 # pano_rgb8_to_mat32f_dev: read_img's image
    want = engine.planet(f32)
    assert gu.same_bits(want, pu.orc_planet(f32))
    coloured = (want[..., 0] >= 0).any()
    assert coloured == (w > 1 and h > 1)
    assert gu.same_bits(engine.planet_pix8(buf, fmt), want), "host entry point"
    assert gu.same_bits(_planet_dev(engine, buf, fmt, w, h), want), "device entry point"


def test_planet_pix8_grey_is_not_divided(engine):
    """Grey pixels are replicated undivided (CImg's spectrum-1 rule) and RGBA's are divided (lodepng's), so the same
    grey values give different planets in the two formats, as read_img gives different images."""
    g = np.random.RandomState(3).randint(0, 256, size=(300, 900)).astype(np.uint8)
    grey = engine.planet_pix8(g, "grey")
    rgba = engine.planet_pix8(xu.to_rgba(np.repeat(g[..., None], 3, axis=2)), "rgba")
    col = grey[..., 0] >= 0
    assert col.any() and grey[col].max() > 1.0 and rgba[col].max() <= 1.0
    assert gu.same_bits(grey, engine.planet(engine.read_img_rgb8(g)))


@pytest.mark.parametrize("fmt", ["rgba", "planar"])
def test_planet_pix8_to_encoder_bytes(engine, fmt):
    """planet_pix8_dev -> pano_mat32f_to_pix8_dev without leaving the device: the buffer write_rgb hands to lodepng
    (RGBA, alpha 255) or CImg (planes) for the planet of read_img's image."""
    buf = _buf(3000, 600, "rgba", seed=11)
    planet = engine.planet(engine.read_img_rgb8(buf, "rgba"))
    want = xu.orc_write_png_rgba(planet) if fmt == "rgba" else xu.orc_write_rgb_planar(planet)
    if xu.have_ref():
        assert np.array_equal(want, xu.ref_write_png(planet) if fmt == "rgba" else xu.ref_write_cimg(planet))
    bpp = 4 if fmt == "rgba" else 3
    d_pix, d_planet = engine.dev_alloc(buf.nbytes), engine.dev_alloc(OUT_BYTES)
    d_out = engine.dev_alloc(pu.SIZE * pu.SIZE * bpp)
    got = np.empty(pu.SIZE * pu.SIZE * bpp, np.uint8)
    try:
        engine.dev_upload(d_pix, buf)
        engine.planet_pix8_dev(d_pix, "rgba", 3000, 600, d_planet)
        engine.mat32f_to_pix8_dev(d_planet, pu.SIZE, pu.SIZE, None, fmt, d_out)
        engine.dev_download(got, d_out)
    finally:
        for d in (d_pix, d_planet, d_out):
            engine.dev_free(d)
    got = got.reshape(want.shape)
    assert np.array_equal(got, want)
    white = (got == 255).all(axis=-1) if fmt == "rgba" else (got == 255).all(axis=0)
    assert white.any() and not white.all()              # the -1 outside the disc turned white, the rest not


@pytest.mark.parametrize("fmt", ["rgb", "rgba", "planar"])
def test_planet_of_strip_mosaic(engine, fmt):
    """The strip pipeline's cropped 8-bit mosaic (mosaic_rgb8_strips) into planet_pix8 equals pano_planet of the
    whole-canvas f32 mosaic after crop, write_rgb's conversion and read_img's."""
    from openpano_b200.stitcher import mosaic_rgb8_strips
    imgs, org = synth.make_stack(6, 260, 200, 90, 17, rows=2, step_y=70)
    items, geom = synth.translation_blend_setup(org, 260, 200)
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    mos = engine.blend([engine.read_img_rgb8(x) for x in pix], items, geom, 0)
    want_rect, want_rgb8 = engine.crop_write_rgb8(mos, crop=True)
    want = engine.planet(engine.read_img_rgb8(want_rgb8))
    assert (want[..., 0] >= 0).any()
    rect, got8 = mosaic_rgb8_strips(engine, items, geom, 0, pix, 37, 2, fmt)
    assert np.array_equal(rect, want_rect)
    assert gu.same_bits(engine.planet_pix8(got8, fmt), want)


def test_planet_pix8_invalid_calls(engine):
    """Null pointers, empty shapes, unknown formats and a misaligned device RGBA source return PANO_ERR_INVALID with
    a message and launch nothing; the context gives correct results afterwards."""
    vp, fp = C.c_void_p, C.POINTER(C.c_float)
    pix = np.zeros(4 * 6 * 4, np.uint8)
    out = np.empty((pu.SIZE, pu.SIZE, 3), np.float32)
    hp, ho = vp(pix.ctypes.data), out.ctypes.data_as(fp)
    d_pix, d_out = engine.dev_alloc(4096), engine.dev_alloc(OUT_BYTES)

    def refused(call, word, what):
        before = engine.launch_count()
        assert call() == -2, what
        assert word in LIB.pano_last_error(engine._h).decode(), what
        assert engine.launch_count() == before, what

    try:
        dp, do = vp(d_pix), vp(d_out)
        assert LIB.pano_planet_pix8(None, hp, PIX_RGB, 6, 4, ho) == -2
        assert LIB.pano_planet_pix8_dev(None, dp, PIX_RGB, 6, 4, do) == -2
        for code in CODE.values():
            refused(lambda: LIB.pano_planet_pix8(engine._h, None, code, 6, 4, ho), "null", ("host pix", code))
            refused(lambda: LIB.pano_planet_pix8(engine._h, hp, code, 6, 4, None), "null", ("host out", code))
            refused(lambda: LIB.pano_planet_pix8_dev(engine._h, None, code, 6, 4, do), "null", ("dev pix", code))
            refused(lambda: LIB.pano_planet_pix8_dev(engine._h, dp, code, 6, 4, None), "null", ("dev out", code))
            for w, h in ((0, 4), (6, 0), (-1, 4), (6, -3)):
                refused(lambda: LIB.pano_planet_pix8(engine._h, hp, code, w, h, ho), "empty", ("host", code, w, h))
                refused(lambda: LIB.pano_planet_pix8_dev(engine._h, dp, code, w, h, do), "empty", ("dev", code, w, h))
        for bad in BAD_FORMATS:
            refused(lambda: LIB.pano_planet_pix8(engine._h, hp, bad, 6, 4, ho), "format", ("host", bad))
            refused(lambda: LIB.pano_planet_pix8_dev(engine._h, dp, bad, 6, 4, do), "format", ("dev", bad))
        for off in (1, 2, 3):
            refused(lambda: LIB.pano_planet_pix8_dev(engine._h, vp(d_pix + off), PIX_RGBA, 6, 4, do), "aligned",
                    ("dev rgba", off))
        # a host RGBA buffer needs no alignment (it is copied to a device block first), nor do the byte layouts
        before = engine.launch_count()
        assert LIB.pano_planet_pix8(engine._h, vp(pix.ctypes.data + 1), PIX_RGBA, 5, 4, ho) == 0
        assert LIB.pano_planet_pix8_dev(engine._h, vp(d_pix + 1), PIX_RGB_PLANAR, 6, 4, do) == 0
        engine.sync()
        assert engine.launch_count() == before + 2
    finally:
        engine.dev_free(d_pix)
        engine.dev_free(d_out)
    with pytest.raises(PanoError):
        engine.planet_pix8(np.zeros((4, 6, 4), np.uint8))         # four channels without fmt="rgba"
    with pytest.raises(PanoError):
        engine.planet_pix8(np.zeros((4, 6, 3), np.uint8), "planar")
    buf = _buf(300, 80, "rgba", seed=5)
    assert gu.same_bits(engine.planet_pix8(buf, "rgba"), pu.orc_planet(engine.read_img_rgb8(buf, "rgba")))


def test_planet_pix8_profile_names(engine):
    """Grey and interleaved RGB run k_planet_rgb8, RGBA and planar k_planet_pix8: one launch per call."""
    try:
        for fmt in FORMATS:
            engine.profile(True)
            engine.profile_reset()
            engine.planet_pix8(_buf(640, 120, fmt, seed=9), fmt)
            engine.sync()
            prof = engine.profile_read()
            want = "k_planet_pix8" if fmt in ("rgba", "planar") else "k_planet_rgb8"
            assert {k: v[0] for k, v in prof.items() if k.startswith("k_planet")} == {want: 1}, (fmt, prof)
    finally:
        engine.profile(False)


def test_cpp_planet_command_equals_reference(tmp_path):
    """load_pixels -> b200_planet -> write_mosaic (openpano_b200/host/pano_host_io.hh) next to the reference's
    write_rgb(IMGFILE(planet), planet(read_img(f))) on PNGs of every colour type, a PPM and a PGM
    (oracle/_ref/planet_pix_test): the written .png and .ppm files byte for byte."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/planet_pix_test not built (needs the reference sources at build time)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(tmp_path)], capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "PLANET PIX TEST OK" in out.stdout
    assert out.stdout.count("identical") == 9 * 2
