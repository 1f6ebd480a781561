"""CPU: the plain-C restatement of the reference's decoder and encoder layouts against the reference's own
read_img / write_rgb with its own lodepng and CImg, bit for bit (oracle/pix_formats.mk builds both).  read_png
meets every PNG colour type through lodepng::decode's RGBA buffer; CImg hands read_img planes; write_rgb writes
lodepng's RGBA for a .png and CImg's planes otherwise.  tests/test_gpu_pixel_formats.py checks the engine
against the same restatement."""
import numpy as np
import pytest

from tests import golden_util as gu
from tests import pix_util as xu
from tests.checker import get_checker

SHAPES = [(2, 2), (3, 50), (50, 3), (37, 29), (64, 48)]   # (w, h)


def _need_ref():
    if not xu.have_ref():
        pytest.skip("oracle/_ref/libopenpano_ref_pix.so not built (needs the reference sources)")


@pytest.mark.parametrize("name", sorted(xu.PNG_CASES))
@pytest.mark.parametrize("w,h", SHAPES)
def test_read_png_every_colour_type(name, w, h):
    _need_ref()
    want, rgba = xu.ref_read_png(name, w, h, seed=w * 31 + h)
    assert gu.same_bits(xu.orc_read_png_rgba(rgba), want)


def test_grey_png_is_divided_unlike_grey_pnm():
    """A grey PNG reaches read_img as RGBA with r = g = b and is divided by 255; the same grey samples through
    CImg (a PGM) are replicated undivided."""
    _need_ref()
    w, h = 40, 30
    png, rgba = xu.ref_read_png("grey", w, h, seed=5)
    raw = xu.png_raw("grey", w, h, seed=5)[0].reshape(h, w)
    assert np.array_equal(rgba[..., 0], raw) and np.array_equal(rgba[..., 1], raw) and np.array_equal(rgba[..., 2], raw)
    pnm, planes = xu.ref_read_cimg(raw)
    assert np.array_equal(planes, raw)
    assert gu.same_bits(pnm, get_checker("orc").read_img_rgb8(raw))
    assert gu.same_bits(png, (raw.astype(np.float64) / 255.0).astype(np.float32)[..., None].repeat(3, 2))
    assert not np.array_equal(png, pnm)


@pytest.mark.parametrize("w,h", SHAPES)
def test_read_cimg_planes(w, h):
    _need_ref()
    rng = np.random.RandomState(w + 100 * h)
    pix = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
    want, planes = xu.ref_read_cimg(pix)
    assert np.array_equal(planes, xu.to_planar(pix))
    assert gu.same_bits(xu.orc_read_img_planar(planes), want)


@pytest.mark.parametrize("w,h", SHAPES)
def test_write_rgb_png_and_cimg(w, h):
    _need_ref()
    mat = xu.mosaic_with_holes(h, w, seed=w * 7 + h)
    assert np.array_equal(xu.orc_write_png_rgba(mat), xu.ref_write_png(mat))
    assert np.array_equal(xu.orc_write_rgb_planar(mat), xu.ref_write_cimg(mat))


def test_layouts_are_relayouts_of_the_interleaved_rules():
    """Without the reference: the new rules are orc_imgio.c's interleaved rules on re-laid-out bytes, and the
    fourth RGBA byte is ignored."""
    orc = get_checker("orc")
    rng = np.random.RandomState(3)
    pix = rng.randint(0, 256, size=(21, 34, 3)).astype(np.uint8)
    want = orc.read_img_rgb8(pix)
    assert gu.same_bits(xu.orc_read_png_rgba(xu.to_rgba(pix, alpha_seed=9)), want)
    assert gu.same_bits(xu.orc_read_img_planar(xu.to_planar(pix)), want)
    mat = xu.mosaic_with_holes(21, 34, seed=4)
    rgb = orc.write_rgb8(mat)
    assert np.array_equal(xu.orc_write_png_rgba(mat), xu.to_rgba(rgb))
    assert np.array_equal(xu.orc_write_rgb_planar(mat), xu.to_planar(rgb))
