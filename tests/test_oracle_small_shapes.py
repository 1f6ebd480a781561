"""CPU: the plain-C oracle against the reference's own translation units at the smallest, thinnest and widest
shapes SIFT, the blenders and the cylinder warp accept, bit for bit.  The inputs are the ones
tests/test_gpu_small_shapes.py runs on the GPU, so the engine-vs-oracle results there are pinned to the
reference too.  Octaves smaller than one 64×32 blur tile or than the blur halo, one-pixel blend ROIs and
warps of sources a few pixels wide are where tile-edge and clamp code runs."""
import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests import golden_util as gu
from tests.test_oracle_vs_ref import _trace_outputs

# ----------------------------------------------------------------------------- SIFT
# (working width, height, NUM_OCTAVE).  The input has the working size itself and SIFT_WORKING_SIZE is
# (w + h) / 2, so the resize ratio is exactly 1.  8 × 300 has the smallest accepted working size and a last
# octave of 6 columns; 11 × 299 and 16 × 16 end on an octave of exactly 6 as well.  Every octave of the
# square cases is smaller than one 64×32 tile, down to 9×9 and 6×6 (smaller than the 13-tap blur window);
# the strips are a few rows or columns high, 8 in their last octave.
SIFT_SHAPES = [(8, 300, 2), (300, 8, 2), (11, 299, 3), (16, 16, 4), (17, 17, 4), (24, 24, 4), (40, 40, 4),
               (64, 32, 4), (65, 33, 4), (72, 48, 4), (1576, 22, 4), (22, 1576, 4), (1548, 50, 4), (50, 1548, 4),
               (1577, 21, 4)]
SIFT_SEEDS = (1, 2, 3)


def sift_noise(w, h, seed):
    """Uniform noise: with both thresholds at 0 it keeps tens of keypoints on images of a few hundred pixels."""
    return np.random.RandomState(1000 * seed + w + 7 * h).rand(h, w, 3).astype(np.float32)


def sift_small_params(w, h, n_oct, **kw):
    assert (w + h) % 2 == 0
    return default_params(sift_working_size=(w + h) // 2, num_octave=n_oct, pre_color_thres=0.0, contrast_thres=0.0, **kw)


def sift_min_desc(w, h):
    """Descriptors every case keeps over its seeds at least (the oracle gives about twice as many)."""
    return 10 if w * h < 2000 else 60


# The full field width: 8191 columns (or rows) with SIFT_WORKING_SIZE 4128 resize by 8256 / 8255, so the
# working image keeps 8191 (the largest accepted) and 64 pixels.
WIDE_SHAPES = [(8191, 64), (64, 8191)]


def wide_input(w, h):
    return synth.make_canvas(h, w, 5), default_params(sift_working_size=4128)


# Other window widths on the tiny shapes: GAUSS_WINDOW_FACTOR 4 and 8 take the generic blur and the full
# extremum scan, DESC_HIST_SCALE_FACTOR 17 and 20 give descriptor windows wider than every octave.
WINDOW_SETS = [("gauss_window_factor", 4), ("gauss_window_factor", 8), ("desc_hist_scale_factor", 17),
               ("desc_hist_scale_factor", 20)]
WINDOW_SHAPES = [(16, 16, 4), (40, 40, 4), (72, 48, 4), (8, 300, 2)]


def sift_trace_outputs(chk, img, p):
    return _trace_outputs(chk.sift_trace(img, p), noct=p.num_octave, nscale=p.num_scale)


# ----------------------------------------------------------------------------- blending
# (source width, height): two, three or a few pixels on one side, narrower or shorter than every multiband
# blur halo (half-widths 6 and 9 at the default window factor).
BLEND_SOURCES = [(3, 50), (50, 3), (2, 2), (12, 7), (130, 20), (9, 300)]
# (bands, GAUSS_WINDOW_FACTOR, LAZY_READ, ORDERED_INPUT); bands 0 is the linear blender.
BLEND_SETS = [(0, 6, 0, 0), (0, 6, 1, 0), (0, 6, 0, 1), (0, 6, 1, 1), (1, 6, 1, 0), (2, 6, 1, 0), (5, 6, 0, 0),
              (2, 4, 1, 0), (5, 4, 1, 0), (2, 8, 0, 0), (5, 8, 1, 0)]


def blend_stack(w, h, seed=3):
    """Three overlapping crops of one canvas, side by side (or stacked for tall sources), and their geometry,
    moved by half a pixel: on whole pixels a 2×2 source is sampled only at column and row 0, where the linear
    blender's weight is 0, and at column 1, where interpolation has no right neighbour."""
    if w >= h:
        imgs, org = synth.make_stack(3, w, h, max(1, w // 2), seed)
    else:
        imgs, org = synth.make_stack(3, w, h, 0, seed, rows=3, step_y=max(1, h // 2))
    items, geom = synth.translation_blend_setup(org, w, h)
    geom["proj_min_x"] += 0.5
    geom["proj_min_y"] += 0.5
    return imgs, items, geom


def one_pixel_stack(seed=4):
    """A 12×7 stack whose first three ROIs are one column (x0 == x1), one row (y0 == y1) and one pixel wide,
    inside the images they sample; the fourth image keeps its whole ROI."""
    imgs, org = synth.make_stack(4, 12, 7, 3, seed)
    items, geom = synth.translation_blend_setup(org, 12, 7)
    geom["proj_min_x"] += 0.5
    geom["proj_min_y"] += 0.5
    x0, y0, x1, y1, hi = items[0]
    xm, ym = (x0 + x1) // 2, (y0 + y1) // 2
    items[0] = (xm, y0, xm, y1, hi)
    x0, y0, x1, y1, hi = items[1]
    xm, ym = (x0 + x1) // 2, (y0 + y1) // 2
    items[1] = (x0, ym, x1, ym, hi)
    x0, y0, x1, y1, hi = items[2]
    xm, ym = (x0 + x1) // 2, (y0 + y1) // 2
    items[2] = (xm, ym, xm, ym, hi)
    return imgs, items, geom


def blend_params(bands, factor, lazy, ordered):
    return default_params(multiband=max(bands, 1), gauss_window_factor=factor, lazy_read=lazy, ordered_input=ordered)


# ----------------------------------------------------------------------------- cylinder warp
WARP_SHAPES = [(3, 50), (50, 3), (7, 5), (65, 33), (4000, 12), (12, 3000)]
WARP_FACTORS = [0.85, 1.0, 1.2]
WARP_FOCALS = [37.0, 10.0]


def warp_input(w, h):
    return synth.make_canvas(h, w, 7 + w + h)


def corner_kpts(w, h):
    """Image-centred keypoints at the four corners, the centre and the middles of two edges."""
    return np.array([[-w / 2, -h / 2], [w / 2, -h / 2], [-w / 2, h / 2], [w / 2, h / 2], [0.0, 0.0],
                     [-w / 2, 0.0], [0.0, h / 2]], np.float64)


# ----------------------------------------------------------------------------- tests
def _same_outputs(got, want):
    assert len(got) == len(want)
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if not gu.same_bits(g, w)]
    assert not bad, f"outputs {bad[:10]} differ from the reference's"


@pytest.mark.parametrize("w,h,n_oct", SIFT_SHAPES)
def test_sift_small_shapes(orc, ref, w, h, n_oct):
    """Every Gaussian and |DoG| plane, the three point stages and the descriptors."""
    p = sift_small_params(w, h, n_oct)
    n_desc = 0
    for seed in SIFT_SEEDS:
        img = sift_noise(w, h, seed)
        got, want = sift_trace_outputs(orc, img, p), sift_trace_outputs(ref, img, p)
        assert tuple(got[0]) == (w, h)
        _same_outputs(got, want)
        n_desc += len(got[-1])
    assert n_desc >= sift_min_desc(w, h), n_desc


@pytest.mark.parametrize("w,h", WIDE_SHAPES)
def test_sift_full_field_width(orc, ref, w, h):
    img, p = wide_input(w, h)
    got, want = sift_trace_outputs(orc, img, p), sift_trace_outputs(ref, img, p)
    assert tuple(got[0]) == (w, h)
    _same_outputs(got, want)
    assert len(got[-1]) > 1000


@pytest.mark.parametrize("field,value", WINDOW_SETS)
@pytest.mark.parametrize("w,h,n_oct", WINDOW_SHAPES)
def test_sift_small_shapes_other_windows(orc, ref, w, h, n_oct, field, value):
    p = sift_small_params(w, h, n_oct, **{field: value})
    for seed in SIFT_SEEDS:
        img = sift_noise(w, h, seed)
        _same_outputs(sift_trace_outputs(orc, img, p), sift_trace_outputs(ref, img, p))


@pytest.mark.parametrize("w,h", BLEND_SOURCES)
def test_blend_small_sources(orc, ref, w, h):
    imgs, items, geom = blend_stack(w, h)
    for s in BLEND_SETS:
        got = orc.blend(imgs, items, geom, s[0], blend_params(*s))
        assert gu.same_bits(got, ref.blend(imgs, items, geom, s[0], blend_params(*s))), s
        if s[0] == 0:
            assert (got[..., 0] >= 0).any(), s


def test_blend_one_pixel_rois(orc, ref):
    imgs, items, geom = one_pixel_stack()
    for s in BLEND_SETS:
        got = orc.blend(imgs, items, geom, s[0], blend_params(*s))
        assert gu.same_bits(got, ref.blend(imgs, items, geom, s[0], blend_params(*s))), s
        assert (got[..., 0] >= 0).any(), s


@pytest.mark.parametrize("focal", WARP_FOCALS)
@pytest.mark.parametrize("w,h", WARP_SHAPES)
def test_cyl_warp_and_crop_small_shapes(orc, ref, w, h, focal):
    img = warp_input(w, h)
    for hf in WARP_FACTORS:
        p = default_params(focal_length=focal)
        assert orc.cyl_warp_shape(w, h, hf, p) == ref.cyl_warp_shape(w, h, hf, p)
        (go, gk), (wo, wk) = orc.cyl_warp(img, corner_kpts(w, h), hf, p), ref.cyl_warp(img, corner_kpts(w, h), hf, p)
        assert go.size and gu.same_bits(go, wo) and gu.same_bits(gk, wk), hf
        (grect, gcrop), (wrect, wcrop) = orc.crop(go), ref.crop(wo)
        assert np.array_equal(grect[2:], wrect[2:]) and gu.same_bits(gcrop, wcrop), hf


def test_cyl_warp_smallest_shapes(orc, ref):
    """A 3×3 image warps to 1×2 pixels, a 2×2 one to none: the reference returns an empty image."""
    for chk in (orc, ref):
        assert chk.cyl_warp_shape(3, 3, 1.0)[:2] == (1, 2)
        assert chk.cyl_warp_shape(2, 2, 1.0)[0] == 0
    img = warp_input(3, 3)
    (go, gk), (wo, wk) = orc.cyl_warp(img, corner_kpts(3, 3)), ref.cyl_warp(img, corner_kpts(3, 3))
    assert gu.same_bits(go, wo) and gu.same_bits(gk, wk)
