"""GPU: the grey plane of every octave, built in one pass over the source image (k_pyramid_grey), against the
oracle bit for bit.  The cases move the tile seams of that pass: working sizes that are or are not tile multiples
(64×32), upscaling resizes, scale factors √2 and 2, 1 to 6 octaves, octaves larger than the working image (their
last rows and columns take the clamped tap si = n - 2 from the last working row / column), 8-bit RGB and grey
sources, and batches of mixed shapes."""
import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests.test_gpu_sift import assert_same, compare_trace

pytestmark = pytest.mark.gpu

# (w, h, params): working size and octave sizes in the comments
CASES = [
    (1500, 1112, {}),                                                   # 918×681: no tile multiple either way
    (600, 400, {}),                                                     # upscaled to 960×640: tile multiples
    (333, 517, dict(scale_factor=2.0, num_scale=6)),                    # upscaled to 626×973, octaves halve
    (640, 480, dict(num_octave=1)),                                     # 914×685, octave 0 only
    (640, 480, dict(num_octave=6)),                                     # down to 162×122
    (800, 600, dict(num_octave=6, scale_factor=2.0, num_scale=6)),      # down to 29×22
    # working size 641×417 (10·64 + 1, 13·32 + 1): the last tile row / column holds one working row / column,
    # and octaves larger than the working image map their last rows and columns to the clamped tap
    (641, 417, dict(sift_working_size=529, scale_factor=0.95, num_octave=3)),
    (641, 417, dict(sift_working_size=529, scale_factor=1.0, num_octave=2)),
]


def _grey_planes(g, o, noct):
    assert g.working_size() == o.working_size()
    assert_same("working", g.plane(0), o.plane(0))
    for oc in range(noct):
        assert g.octave_size(oc) == o.octave_size(oc)
        assert_same(f"grey[{oc}]", g.plane(1, oc, 0), o.plane(1, oc, 0))


@pytest.mark.parametrize("w,h,kw", CASES)
def test_octave_grey_planes_bit_exact(engine, orc, w, h, kw):
    p = default_params(**kw)
    img = synth.make_canvas(h, w, w + h)
    g, o = engine.sift_trace(img, p), orc.sift_trace(img, p)
    try:
        _grey_planes(g, o, p.num_octave)
        n = compare_trace(g, o, nscale=p.num_scale, noct=p.num_octave)
        if p.scale_factor > 1:
            assert n > 100
    finally:
        g.close()
        o.close()


def _same_features(fs, want):
    try:
        for i, (co, do) in enumerate(want):
            c, d = fs.download(i)
            assert_same(f"coor[{i}]", c, co)
            assert_same(f"desc[{i}]", d, do)
    finally:
        fs.free()


@pytest.mark.parametrize("kw", [{}, dict(num_octave=6), dict(scale_factor=2.0, num_scale=6)])
def test_mixed_batch(engine, orc, kw):
    """One f32 batch of shapes that up- and downscale, with and without tile multiples."""
    p = default_params(**kw)
    imgs = [synth.make_canvas(h, w, 3 * w + h) for w, h in ((1500, 1112), (600, 400), (333, 517), (641, 417))]
    _same_features(engine.sift_detect_batch(imgs, p), [orc.sift_detect(im, p) for im in imgs])


@pytest.mark.parametrize("kw", [{}, dict(num_octave=6), dict(scale_factor=2.0, num_scale=6)])
def test_rgb8_sources(engine, orc, kw):
    """8-bit RGB and grey sources in one batch: the features of read_img's f32 images."""
    p = default_params(**kw)
    pix = []
    for k, (w, h) in enumerate(((1500, 1112), (600, 400), (333, 517), (1300, 867))):
        x = (synth.make_canvas(h, w, 5 * w + h) * 255.0 + 0.5).astype(np.uint8)
        pix.append(x if k % 2 == 0 else np.ascontiguousarray(x[..., 1]))
    want = [orc.sift_detect(orc.read_img_rgb8(x), p) for x in pix]
    assert min(len(d) for _, d in want) > 100
    _same_features(engine.sift_detect_batch_rgb8(pix, p), want)
