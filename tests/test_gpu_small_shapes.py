"""GPU: SIFT, both blenders and the cylinder warp at the smallest, thinnest and widest shapes they accept, bit for
bit against the oracle (pinned to the reference at the same inputs in tests/test_oracle_small_shapes.py), and the
shape limits on both sides.  The image kernels cut planes into 64×32 tiles with halos; here octaves and ROIs are
smaller than one tile or one blur halo, so a tile's edge fill happens on both of its sides, every extremum
candidate sits on a tile seam, and candidate keys reach the last of their 13-bit columns and rows."""
import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests import golden_util as gu
from tests.test_gpu_rgb8_warp_strips import _Dev, _strips_both, _warp_both
from tests.test_gpu_sift import assert_same, compare_trace
from tests.test_oracle_small_shapes import (BLEND_SETS, BLEND_SOURCES, SIFT_SEEDS, SIFT_SHAPES, WARP_FACTORS, WARP_FOCALS,
                                            WARP_SHAPES, WIDE_SHAPES, WINDOW_SETS, WINDOW_SHAPES, blend_params, blend_stack,
                                            corner_kpts, one_pixel_stack, sift_min_desc, sift_noise, sift_small_params,
                                            warp_input, wide_input)

pytestmark = pytest.mark.gpu
PANO_ERR_INVALID = -2


# ----------------------------------------------------------------------------- SIFT
def _trace_case(engine, orc, img, p):
    g, o = engine.sift_trace(img, p), orc.sift_trace(img, p)
    try:
        assert g.working_size() == o.working_size()
        return compare_trace(g, o, nscale=p.num_scale, noct=p.num_octave)
    finally:
        g.close()
        o.close()


@pytest.mark.parametrize("w,h,n_oct", SIFT_SHAPES)
def test_sift_trace_small_shapes(engine, orc, w, h, n_oct):
    p = sift_small_params(w, h, n_oct)
    n = 0
    for seed in SIFT_SEEDS:
        img = sift_noise(w, h, seed)
        n += _trace_case(engine, orc, img, p)
    assert n >= sift_min_desc(w, h), n


@pytest.mark.parametrize("w,h", WIDE_SHAPES)
def test_sift_trace_full_field_width(engine, orc, w, h):
    """Working images 8191 wide or tall: candidate keys carry x (or y) up to 8190 in their 13-bit fields."""
    img, p = wide_input(w, h)
    g, o = engine.sift_trace(img, p), orc.sift_trace(img, p)
    try:
        assert g.working_size() == (w, h)
        far = o.points(0)["x" if w > h else "y"]
        assert (far > 8000).any(), far.max()
        assert compare_trace(g, o) > 1000
    finally:
        g.close()
        o.close()


@pytest.mark.parametrize("field,value", WINDOW_SETS)
@pytest.mark.parametrize("w,h,n_oct", WINDOW_SHAPES)
def test_sift_trace_small_shapes_other_windows(engine, orc, w, h, n_oct, field, value):
    p = sift_small_params(w, h, n_oct, **{field: value})
    n = sum(_trace_case(engine, orc, sift_noise(w, h, seed), p) for seed in SIFT_SEEDS)
    assert n >= 3, n      # the 13- and 25-tap windows of factor 8 keep 4 descriptors on 16×16


# Ragged batches: (SIFT_WORKING_SIZE, NUM_OCTAVE, input shapes).  Every shape of a batch has w + h equal to
# twice the working size, so each image keeps its shape.
SIFT_BATCHES = [(154, 2, [(8, 300), (300, 8), (150, 158), (11, 297)]),
                (24, 4, [(24, 24), (16, 32), (32, 16), (17, 31)]),
                (48, 4, [(64, 32), (32, 64), (48, 48), (65, 31)]),
                (799, 4, [(1576, 22), (22, 1576), (1548, 50), (50, 1548), (1577, 21)])]


def _batch_params(ws, n_oct):
    return default_params(sift_working_size=ws, num_octave=n_oct, pre_color_thres=0.0, contrast_thres=0.0)


@pytest.mark.parametrize("ws,n_oct,shapes", SIFT_BATCHES)
def test_sift_batch_small_shapes(engine, orc, ws, n_oct, shapes):
    p = _batch_params(ws, n_oct)
    imgs = [sift_noise(w, h, 4) for w, h in shapes]
    fs = engine.sift_detect_batch(imgs, p)
    n = 0
    try:
        for i, im in enumerate(imgs):
            c, d = fs.download(i)
            co, do = orc.sift_detect(im, p)
            assert_same(f"coor[{i}]", c, co)
            assert_same(f"desc[{i}]", d, do)
            n += len(d)
    finally:
        fs.free()
    assert n >= 10 * len(shapes), n


@pytest.mark.parametrize("ws,n_oct,shapes", SIFT_BATCHES)
def test_sift_batch_rgb8_small_shapes(engine, orc, ws, n_oct, shapes):
    """8-bit sources, colour and grey in turn, against the oracle on read_img's f32 images of the same pixels."""
    p = _batch_params(ws, n_oct)
    rng = np.random.RandomState(ws)
    pix = [rng.randint(0, 256, (h, w, 3) if k % 2 == 0 else (h, w)).astype(np.uint8) for k, (w, h) in enumerate(shapes)]
    fs = engine.sift_detect_batch_rgb8(pix, p)
    n = 0
    try:
        for i, x in enumerate(pix):
            c, d = fs.download(i)
            co, do = orc.sift_detect(orc.read_img_rgb8(x), p)
            assert_same(f"coor[{i}]", c, co)
            assert_same(f"desc[{i}]", d, do)
            n += len(d)
    finally:
        fs.free()
    assert n >= 10 * len(shapes), n


# ----------------------------------------------------------------------------- blending
BLEND_STACKS = [(f"{w}x{h}", lambda w=w, h=h: blend_stack(w, h)) for w, h in BLEND_SOURCES] + [("one_pixel", one_pixel_stack)]


def _covered(mosaic):
    return (mosaic[..., 0] >= 0).any()


@pytest.mark.parametrize("name,stack", BLEND_STACKS, ids=[n for n, _ in BLEND_STACKS])
def test_blend_small_sources(engine, orc, name, stack):
    imgs, items, geom = stack()
    for s in BLEND_SETS:
        p = blend_params(*s)
        got = engine.blend(imgs, items, geom, s[0], p)
        assert gu.same_bits(got, orc.blend(imgs, items, geom, s[0], p)), (name, s)
        if s[0] == 0:
            assert _covered(got), (name, s)


def _rows_f32(engine, imgs, items, geom, bands, p, cuts):
    """(pano_blend_dev, the strips of pano_blend_rows_dev between consecutive cuts), from f32 device sources."""
    shapes = [im.shape[:2] for im in imgs]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    dev = _Dev(engine)
    try:
        d_src = [dev.upload(im) for im in imgs]
        d_out = dev.alloc(tw * th * 12)
        full = np.empty((th, tw, 3), np.float32)
        engine.blend_dev(d_src, shapes, items, geom, d_out, tw, th, bands, p)
        engine.dev_download(full, d_out)
        parts = []
        for r0, r1 in zip(cuts[:-1], cuts[1:]):
            part = np.empty((r1 - r0, tw, 3), np.float32)
            engine.blend_rows_dev(d_src, shapes, items, geom, d_out, tw, th, r0, r1, bands, p)
            engine.dev_download(part, d_out)
            parts.append(part)
    finally:
        dev.free()
    return full, parts


ROW_STACKS = [("50x3", lambda: blend_stack(50, 3)), ("130x20", lambda: blend_stack(130, 20)),
              ("12x7", lambda: blend_stack(12, 7)), ("one_pixel", one_pixel_stack)]
ROW_SETS = [(0, 6, 0, 0), (0, 6, 1, 1), (2, 6, 1, 0), (5, 6, 0, 0), (5, 4, 1, 0)]


@pytest.mark.parametrize("name,stack", ROW_STACKS, ids=[n for n, _ in ROW_STACKS])
def test_blend_rows_of_small_canvases(engine, orc, name, stack):
    """Strips of one row and strips thinner than the multiband halo, concatenated: pano_blend_dev's mosaic."""
    imgs, items, geom = stack()
    th = max(it[3] for it in items)
    cuts = list(range(th + 1)) if th <= 12 else [0, 1, 2, 3, 7, 8, 8, 13, th]
    for s in ROW_SETS:
        p = blend_params(*s)
        full, parts = _rows_f32(engine, imgs, items, geom, s[0], p, cuts)
        assert gu.same_bits(full, orc.blend(imgs, items, geom, s[0], p)), (name, s)
        assert gu.same_bits(np.concatenate(parts), full), (name, s)
        if s[0] == 0:
            assert _covered(full), (name, s)


def test_blend_stream_and_rgb8_small_sources(engine, orc):
    """One case each through the blend stream and pano_blend_rgb8_dev (with its row strips)."""
    imgs, items, geom = blend_stack(50, 3)
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    pix[1] = np.ascontiguousarray(pix[1][..., 0])
    f32 = [orc.read_img_rgb8(x) for x in pix]
    th = max(it[3] for it in items)
    for bands in (0, 5):
        p = blend_params(bands, 6, 1, 0)
        want = orc.blend(f32, items, geom, bands, p)
        assert gu.same_bits(engine.blend_lazy(pix, items, geom, bands, p, window=1), want), bands
        conv, full, parts = _strips_both(engine, pix, items, geom, bands, p, list(range(th + 1)))
        assert gu.same_bits(conv, want) and gu.same_bits(full, want), bands
        assert gu.same_bits(np.concatenate(parts), want), bands


# ----------------------------------------------------------------------------- cylinder warp
@pytest.mark.parametrize("focal", WARP_FOCALS)
@pytest.mark.parametrize("w,h", WARP_SHAPES)
def test_cyl_warp_small_shapes(engine, orc, w, h, focal):
    """pano_cyl_warp, pano_cyl_warp_batch_dev and pano_cyl_warp_batch_rgb8_dev (one and three channels) with
    keypoints at the image corners."""
    img = warp_input(w, h)
    pix3 = (img * 255.0 + 0.5).astype(np.uint8)
    pix = [pix3, np.ascontiguousarray(pix3[..., 2])]
    for hf in WARP_FACTORS:
        p = default_params(focal_length=focal)
        o_img, o_kp = orc.cyl_warp(img, corner_kpts(w, h), hf, p)
        g_img, g_kp = engine.cyl_warp(img, corner_kpts(w, h), hf, p)
        assert o_img.size and gu.same_bits(g_img, o_img) and gu.same_bits(g_kp, o_kp), hf
        kpts = [corner_kpts(w, h) for _ in pix]
        want, got, ka, kb = _warp_both(engine, pix, hf, kpts, p)
        for k, x in enumerate(pix):
            r_img, r_kp = orc.cyl_warp(orc.read_img_rgb8(x), corner_kpts(w, h), hf, p)
            assert gu.same_bits(want[k], r_img) and gu.same_bits(got[k], r_img), (hf, k)
            assert gu.same_bits(ka[k], r_kp) and gu.same_bits(kb[k], r_kp), (hf, k)


# ----------------------------------------------------------------------------- limits
def _refused(engine, call, words):
    """call() must fail with PANO_ERR_INVALID and a message naming the limit, before any kernel launch."""
    from openpano_b200.capi import PanoError
    before = engine.launch_count()
    with pytest.raises(PanoError) as ei:
        call()
    assert ei.value.code == PANO_ERR_INVALID
    assert words in str(ei.value), str(ei.value)
    assert engine.launch_count() == before


def _sift_matches_oracle(engine, orc, img, p):
    c, d = engine.sift_detect(img, p)
    co, do = orc.sift_detect(img, p)
    assert_same("coor", c, co)
    assert_same("desc", d, do)
    return len(d)


def test_sift_working_size_limits(engine, orc):
    """Working sizes 8 and 8191 are accepted (8191 in test_sift_trace_full_field_width), 7 and 8192 refused;
    inputs of w + h = 2 × SIFT_WORKING_SIZE keep their size."""
    for w, h, ws in ((7, 299, 153), (299, 7, 153), (8192, 64, 4128), (64, 8192, 4128)):
        img = np.random.RandomState(w).rand(h, w, 3).astype(np.float32)
        _refused(engine, lambda: engine.sift_detect(img, default_params(sift_working_size=ws, num_octave=1)),
                 "working size")
        n = 0
        for w2, h2 in ((8, 300), (300, 8)):
            n += _sift_matches_oracle(engine, orc, sift_noise(w2, h2, 5), sift_small_params(w2, h2, 2))
        assert n > 0


def test_sift_last_octave_limit(engine, orc):
    """A last octave of 6 pixels is accepted (16×16 over four octaves: 16, 12, 8, 6), one of 5 refused (14×14:
    14, 10, 7, 5)."""
    img = sift_noise(14, 14, 1)
    _refused(engine, lambda: engine.sift_detect(img, sift_small_params(14, 14, 4)), "octave too small")
    n = sum(_sift_matches_oracle(engine, orc, sift_noise(16, 16, s), sift_small_params(16, 16, 4)) for s in SIFT_SEEDS)
    assert n > 0


def test_blend_source_limit(engine, orc):
    """Blend sources 2 pixels wide and high are accepted, 1 pixel wide or high refused."""
    imgs, items, geom = blend_stack(2, 2)
    for shape in ((2, 1, 3), (1, 2, 3)):
        bad = list(imgs)
        bad[1] = np.ascontiguousarray(np.resize(imgs[1], shape))
        for bands in (0, 2):
            _refused(engine, lambda: engine.blend(bad, items, geom, bands, blend_params(bands, 6, 1, 0)), "invalid shape")
        for bands in (0, 2):
            p = blend_params(bands, 6, 1, 0)
            got = engine.blend(imgs, items, geom, bands, p)
            assert gu.same_bits(got, orc.blend(imgs, items, geom, bands, p)) and _covered(got), bands


def test_cyl_warp_empty_limit(engine, orc):
    """The warp of a 3×3 image (1×2 pixels) is accepted; that of a 2×2 image is 0 pixels wide and refused."""
    assert engine.cyl_warp_shape(2, 2)[0] == 0 and engine.cyl_warp_shape(3, 3)[:2] == (1, 2)
    small, tiny = warp_input(3, 3), warp_input(2, 2)
    _refused(engine, lambda: engine.cyl_warp(tiny, corner_kpts(2, 2)), "warp is 0x1")
    dev = _Dev(engine)
    try:
        d_src, d_out = dev.upload(tiny), dev.alloc(256)
        _refused(engine, lambda: engine.cyl_warp_batch_dev([d_src], [(2, 2)], [d_out], [corner_kpts(2, 2)]), "warp is 0x1")
        d_pix = dev.upload((tiny * 255.0).astype(np.uint8))
        _refused(engine, lambda: engine.cyl_warp_batch_rgb8_dev([d_pix], [3], [(2, 2)], [d_out], None), "warp is 0x1")
    finally:
        dev.free()
    o_img, o_kp = orc.cyl_warp(small, corner_kpts(3, 3))
    g_img, g_kp = engine.cyl_warp(small, corner_kpts(3, 3))
    assert gu.same_bits(g_img, o_img) and gu.same_bits(g_kp, o_kp) and _covered(g_img)
