"""CPU: the plain-C oracle against the reference's own blender and encoder translation units, bit for bit, where
the blend's inverse map reaches the lens horizon (360° canvases, wide flat yaw, adversarial inverse maps: see
tests/wide_geometry.py) and where write_rgb's float -> u8 truncation leaves [0, 255].

Both sides convert with x86-64's cvttss2si / cvttsd2si, which gives INT_MIN for NaN and for anything outside
[-2^31, 2^31): a NaN, infinite or >= 2^31 coordinate floors to INT_MIN and interpolate() returns Color::NO, and a
product (v < 0 ? 1 : v) * 255 that is NaN, +inf or >= 2^31 encodes as 0.  These tests pin that behaviour, which the
engine's kernels must reproduce (tests/test_gpu_wide_geometry.py)."""
import numpy as np
import pytest

from openpano_b200._abi import default_params
from tests import golden_util as gu
from tests import pix_util as xu
from tests import wide_geometry as wg

LINEAR = [(0, 0), (0, 1), (1, 0), (1, 1)]      # (lazy_read, ordered_input)


def _blend_both(orc, ref, name, bands, lazy=1, ordered=0):
    imgs, items, geom = wg.geometry(name)
    p = default_params(lazy_read=lazy, ordered_input=ordered, multiband=bands)
    want = ref.blend(imgs, items, geom, bands, p)
    got = orc.blend(imgs, items, geom, bands, p)
    assert gu.same_bits(got, want), (name, bands, lazy, ordered)
    assert not np.isnan(want).any()               # a NaN coordinate is Color::NO, never a NaN pixel
    return want


@pytest.mark.parametrize("name", wg.GEOMETRIES)
def test_linear_blend_at_lens_horizon(orc, ref, name):
    outs = [_blend_both(orc, ref, name, 0, lazy, ordered) for lazy, ordered in LINEAR]
    assert (outs[0][..., 0] >= 0).mean() > 0.15, name


@pytest.mark.parametrize("bands", [1, 3])
@pytest.mark.parametrize("name", wg.GEOMETRIES)
def test_multiband_blend_at_lens_horizon(orc, ref, name, bands):
    out = _blend_both(orc, ref, name, bands)
    assert (out[..., 0] >= 0).mean() > 0.15, name


def test_rigs_reach_the_lens_horizon():
    """In every rig some image's ROI holds canvas pixels on both sides of its lens horizon (rz of both signs along
    the ROI's middle row); in the 360° rigs that is an image whose ROI spans the whole canvas width.  Without that
    the rigs would test nothing new."""
    for name in wg.RIGS:
        imgs, items, geom = wg.geometry(name)
        tw = max(it[2] for it in items)
        crossing = []
        for x0, y0, x1, y1, hi in items:
            hi = np.array(hi).reshape(3, 3)
            cx = np.arange(x0, x1 + 1) * geom["res_x"] + geom["proj_min_x"]
            cy = (y0 + y1) // 2 * geom["res_y"] + geom["proj_min_y"]
            if geom["projection"] == 0:
                h = np.stack([cx, np.full_like(cx, cy), np.ones_like(cx)])
            else:
                h = np.stack([np.sin(cx), np.full_like(cx, cy if geom["projection"] == 1 else np.tan(cy)), np.cos(cx)])
            rz = hi[2] @ h
            if (rz < 0).any() and (rz > 0).any():
                crossing.append((x0, x1))
        assert crossing, name
        if geom["projection"] != 0:
            assert any(x0 == 0 and x1 >= tw - 1 for x0, x1 in crossing), name


def test_u8_sweep_model_is_x86():
    """The numpy model of write_rgb's conversion, on the values where it matters."""
    v = np.array([np.inf, np.nan, 2.0 ** 31 / 255 * 1.0001, 255.9 / 255, 256 / 255, 1.0, -0.0, -np.inf, -1e-45],
                 np.float32)
    assert list(wg.x86_write_rgb(v)) == [0, 0, 0, 255, 0, 255, 0, 255, 255]


def test_u8_sweep_write_rgb(orc, ref):
    """orc_write_rgb8 against the reference's write_rgb (PNM through CImg) and the x86 model."""
    m = wg.u8_sweep_mosaic()
    want = ref.write_rgb8(m)
    assert np.array_equal(want, wg.x86_write_rgb(m))
    assert np.array_equal(orc.write_rgb8(m), want)


def test_u8_sweep_encoder_layouts():
    """write_png's RGBA buffer and write_rgb's CImg planes (oracle/pix_formats.mk) on the sweep."""
    if not xu.have_ref():
        pytest.skip("oracle/_ref/libopenpano_ref_pix.so not built (needs the reference sources)")
    m = wg.u8_sweep_mosaic()
    rgb = wg.x86_write_rgb(m)
    want_png, want_cimg = xu.ref_write_png(m), xu.ref_write_cimg(m)
    assert np.array_equal(want_png, xu.to_rgba(rgb)) and np.array_equal(want_cimg, xu.to_planar(rgb))
    assert np.array_equal(xu.orc_write_png_rgba(m), want_png)
    assert np.array_equal(xu.orc_write_rgb_planar(m), want_cimg)
