"""GPU: the cylinder sweep (pano_blend_sweep_create_cyl, stitcher.cylinder_mosaic_rgb8_sweep).  Its bytes and
rectangle must equal write_rgb(crop(perspective_correction(blend))) — the cylinder stream's whole f32 mosaic, the
plain-C correction pass (oracle/orc_persp.c, pinned to the reference by tests/test_oracle_persp.py), then crop and
write_rgb's conversion — for both blenders, both LAZY_READ branches, strip heights from 1 row to the whole canvas,
keep budgets from none to unlimited, f32 and 8-bit sources in every PANO_PIX_* format on the host and the device,
every output layout with crop on and off, and config 1's shape against the oracle's warp + blend.  Its hand-overs must
be the plan's, and misuse must be sticky."""
import ctypes as C

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from openpano_b200.capi import (PIX_FORMATS, SIZE_MAX, SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_DEV, SRC_RGB8_HOST, Engine,
                                PanoError, blend_sweep_plan_cyl)
from openpano_b200.stitcher import cylinder_mosaic_rgb8_sweep
from tests import golden_util as gu
from tests import persp_util as pu
from tests.test_gpu_blend_cyl import _case, _code, _layout, _stream

pytestmark = pytest.mark.gpu


def _src_shapes(srcs, fmts):
    return [s.shape[1:] if f == "planar" else s.shape[:2] for s, f in zip(srcs, fmts)]


def _want(engine, mosaic, inv, params, crop, out):
    """write_rgb(crop(perspective_correction(mosaic))) of an f32 mosaic: the oracle's correction pass, then the
    engine's whole-canvas crop and conversion."""
    corrected = pu.orc_correct(mosaic, inv, params.lazy_read, params.ordered_input)
    return engine.crop_write_pix8(corrected, crop, out)


def _sweep(engine, items, geom, inv, bands, srcs, fmts, rows, keep, out="rgb", crop=True, params=None, **kw):
    st = {}
    if "kind" not in kw:
        kw["fmt"] = None if fmts[0] == "f32" else fmts
    rect, px = cylinder_mosaic_rgb8_sweep(engine, items, geom, 1.0, inv, bands, srcs, rows, keep, out, crop, params,
                                          stats=st, **kw)
    return rect, px, st


def _check(engine, items, geom, inv, bands, srcs, fmts, rows, keep, want, out="rgb", crop=True, params=None, **kw):
    rect, px, st = _sweep(engine, items, geom, inv, bands, srcs, fmts, rows, keep, out, crop, params, **kw)
    want_rect, want_px = want
    assert (rect is None) == (not crop)
    if crop:
        assert np.array_equal(rect, want_rect), (rows, keep)
    assert gu.same_bits(px, want_px), (rows, keep, out, crop)
    return st


def _keeps(shapes, items, geom, bands, inv, rows, nbytes):
    live = blend_sweep_plan_cyl(shapes, items, geom, bands, inv, rows, nbytes, SIZE_MAX)["retained_high"]
    return [0, live, SIZE_MAX]


@pytest.mark.parametrize("lazy", [1, 0])
@pytest.mark.parametrize("bands", [0, 2, 5])
@pytest.mark.parametrize("name", ["random", "keystone", "z_cross"])
def test_sweep_equals_whole_canvas_chain(engine, name, bands, lazy):
    """8-bit RGB host sources; strips of 1, 21, 256 rows and the whole canvas; keep 0, the largest kept set and
    unlimited; the hand-overs are the plan's."""
    p = default_params(lazy_read=lazy)
    rgb, items, geom = _case(n=6, params=p)
    shapes = [x.shape[:2] for x in rgb]
    mosaic = _stream(engine, rgb, ["rgb"] * 6, items, geom, bands, 1.0, [6], p)
    oh, ow = mosaic.shape[:2]
    inv = pu.inv_cases(ow, oh, seed=bands)[name]
    want = _want(engine, mosaic, inv, p, True, "rgb")
    nbytes = [x.nbytes for x in rgb]
    for rows in (1, 21, 256, oh):
        for keep in _keeps(shapes, items, geom, bands, inv, rows, nbytes):
            st = _check(engine, items, geom, inv, bands, rgb, ["rgb"] * 6, rows, keep, want, params=p)
            pl = blend_sweep_plan_cyl(shapes, items, geom, bands, inv, rows, nbytes, keep, p)
            assert (st["uploads"], st["upload_bytes"], st["retained_high"]) == \
                (pl["n_uploads"], pl["upload_bytes"], pl["retained_high"]), (rows, keep)
            if keep == SIZE_MAX:
                assert st["upload_bytes"] == sum(nbytes)


@pytest.mark.parametrize("fmt", ["grey", "rgb", "rgba", "planar", "f32"])
def test_every_format_layout_and_crop(engine, fmt):
    rgb, items, geom = _case(n=5)
    srcs = [_layout(x, fmt) for x in rgb]
    fmts = [fmt] * 5
    p = default_params()
    mosaic = _stream(engine, srcs, fmts, items, geom, 0, 1.0, [5], p)
    oh, ow = mosaic.shape[:2]
    inv = pu.inv_cases(ow, oh, seed=4)["keystone"]
    for out, crop in (("rgb", True), ("rgba", False), ("planar", True), ("rgb", False)):
        want = _want(engine, mosaic, inv, p, crop, out)
        _check(engine, items, geom, inv, 0, srcs, fmts, 37, SIZE_MAX, want, out, crop)


@pytest.mark.parametrize("kind", ["rgb8_host", "rgb8_dev", "f32_host", "f32_dev"])
@pytest.mark.parametrize("bands", [0, 2])
def test_pointer_source_kinds(engine, kind, bands):
    """Pinned host and device sources, f32 and 8-bit in mixed PANO_PIX_* formats."""
    rgb, items, geom = _case(n=8)
    fmts8 = ["rgb", "grey", "rgba", "planar"] * 2
    u8 = kind.startswith("rgb8")
    srcs = [_layout(x, f) for x, f in zip(rgb, fmts8)] if u8 else [_layout(x, "f32") for x in rgb]
    fmts = fmts8 if u8 else ["f32"] * 8
    mosaic = _stream(engine, srcs, fmts, items, geom, bands, 1.0, [1] * 8)
    oh, ow = mosaic.shape[:2]
    inv = pu.inv_cases(ow, oh, seed=7)["random"]
    want = _want(engine, mosaic, inv, default_params(), True, "planar")
    code = {"rgb8_host": SRC_RGB8_HOST, "rgb8_dev": SRC_RGB8_DEV, "f32_host": SRC_F32_HOST, "f32_dev": SRC_F32_DEV}[kind]
    host = code in (SRC_RGB8_HOST, SRC_F32_HOST)
    ptrs = [Engine.host_alloc(x.nbytes) if host else engine.dev_alloc(x.nbytes) for x in srcs]
    try:
        for q, x in zip(ptrs, srcs):
            if host:
                C.memmove(q, x.ctypes.data, x.nbytes)
            else:
                engine.dev_upload(q, x)
        shapes = _src_shapes(srcs, fmts)
        codes = [_code(f) for f in fmts]
        nbytes = [x.nbytes for x in srcs]
        for rows in (1, 33):
            for keep in _keeps(shapes, items, geom, bands, inv, rows, nbytes):
                _check(engine, items, geom, inv, bands, ptrs, fmts, rows, keep, want, "planar", True, kind=code,
                       formats=codes, shapes=shapes)
    finally:
        for q in ptrs:
            Engine.host_free(q) if host else engine.dev_free(q)


def test_config1_against_the_oracle(engine, orc):
    """BASELINE config 1 (CMU0, cylinder mode) at its shape: the sweep on the 8-bit sources equals the oracle's warp
    of every read_img image, LinearBlender over the warped images, the correction pass, crop and write_rgb."""
    from tests.checker import get_checker
    omt = get_checker("orc_mt")
    views, org = synth.config_stack("cmu0_8x600x400")
    pix = [(v * 255.0 + 0.5).astype(np.uint8) for v in views]
    imgs = [orc.read_img_rgb8(x) for x in pix]
    h, w = imgs[0].shape[:2]
    params = default_params(ordered_input=1)
    ow, oh, _, _ = engine.cyl_warp_shape(w, h, 1.0, params)
    warped = [orc.cyl_warp(im, np.zeros((0, 2)), 1.0, params)[0] for im in imgs]
    items, geom = synth.translation_blend_setup(org, ow, oh)
    mosaic = omt.blend(warped, items, geom, 0, params)
    mh, mw = mosaic.shape[:2]
    inv = pu.keystone(mw, mh, 0.08, 0.0, 0.02)
    corrected = pu.orc_correct(mosaic, inv, params.lazy_read, params.ordered_input)
    want_rect, cropped = orc.crop(corrected)
    want_px = orc.write_rgb8(cropped)
    for rows in (256, mh):
        rect, px, _ = _sweep(engine, items, geom, inv, 0, pix, ["rgb"] * len(pix), rows, SIZE_MAX, params=params)
        assert np.array_equal(rect[2:], want_rect[2:]), (rect, want_rect)
        assert gu.same_bits(px.reshape(want_px.shape), want_px), rows


def test_golden_fixture(engine):
    """The reference's corrected mosaics of a small cylinder stack (tests/golden/cyl_persp.npz), through the sweep
    from the fixture's 8-bit sources, uncropped."""
    g = gu.load("cyl_persp.npz")
    pix = list(g["pix"])
    mn = g["geom_min"]
    items = [tuple(int(v) for v in b) + (list(hi),) for b, hi in zip(g["items_box"], g["items_inv"])]
    geom = dict(projection=0, res_x=1.0, res_y=1.0, proj_min_x=float(mn[0]), proj_min_y=float(mn[1]))
    p = default_params(lazy_read=int(g["lazy"]), ordered_input=int(g["ordered"]))
    for key in ("mild", "keystone"):
        want = engine.crop_write_pix8(g[f"{key}_want"], False, "rgb")
        for rows in (1, 21):
            _check(engine, items, geom, g[f"{key}_inv"], 0, pix, ["rgb"] * 3, rows, 0, want, "rgb", False, p)


def test_misuse_is_invalid_and_sticky(engine):
    from openpano_b200.capi import LIB
    rgb, items, geom = _case(n=4)
    h, w = rgb[0].shape[:2]
    p = default_params()
    ow, oh, _, _ = Engine.cyl_warp_shape(w, h, 1.0, p)
    arr, g = engine._blend_args([None] * 4, [(oh, ow)] * 4, items, geom)
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    sw, sh = (C.c_int * 4)(*[w] * 4), (C.c_int * 4)(*[h] * 4)
    inv = (C.c_double * 9)(*np.eye(3).ravel())
    hnd = C.c_void_p()
    create = LIB.pano_blend_sweep_create_cyl

    def make(**kw):
        a = dict(ctx=engine._h, n=4, imgs=arr, sw=sw, sh=sh, inv=inv, tw=tw, rows=16, out=C.byref(hnd))
        a.update(kw)
        return create(a["ctx"], a["n"], a["imgs"], a["sw"], a["sh"], 1.0, C.byref(g), 0, C.byref(p), a["tw"], th,
                      a["inv"], a["rows"], None, SIZE_MAX, 1, a["out"])

    assert make() == 0
    LIB.pano_blend_sweep_free(hnd)
    one = (C.c_int * 4)(1, w, w, w)
    for name, kw in {"null inv": dict(inv=None), "null widths": dict(sw=None), "source under 2x2": dict(sw=one),
                     "no strip rows": dict(rows=0), "wrong canvas": dict(tw=tw + 1), "null out": dict(out=None),
                     "null ctx": dict(ctx=None), "no images": dict(n=0)}.items():
        assert make(**kw) == -2, name
    bad, _ = engine._blend_args([None] * 4, [(oh + 1, ow)] + [(oh, ow)] * 3, items, geom)
    assert make(imgs=bad) == -2
    assert "warps to" in LIB.pano_last_error(engine._h).decode()
    # misuse of the handle: a strip missing a source, then every call returns the same failure
    s = engine.blend_sweep_cyl([(h, w)] * 4, items, geom, 1.0, np.eye(3), 16, SIZE_MAX)
    try:
        st, want = s.next()
        assert st == 0 and want.any()
        with pytest.raises(PanoError) as ei:
            s.strip([0] * 4, [3] * 4, SRC_RGB8_HOST)
        assert ei.value.code == -2
        with pytest.raises(PanoError):
            s.strip([x.ctypes.data if k else 0 for x, k in zip(rgb, want)], [3] * 4, SRC_RGB8_HOST)
        with pytest.raises(PanoError):
            s.next()
    finally:
        s.close()
    # the context is still usable
    mosaic = _stream(engine, rgb, ["rgb"] * 4, items, geom, 0, 1.0, [4], p)
    want = _want(engine, mosaic, np.eye(3), p, True, "rgb")
    _check(engine, items, geom, np.eye(3), 0, rgb, ["rgb"] * 4, 16, SIZE_MAX, want)


def test_profile_name(engine):
    rgb, items, geom = _case(n=4)
    engine.profile(True)
    engine.profile_reset()
    try:
        _sweep(engine, items, geom, np.eye(3), 0, rgb, ["rgb"] * 4, 64, SIZE_MAX)
        prof = engine.profile_read()
    finally:
        engine.profile(False)
    oh = max(it[3] for it in items)
    assert prof.get("k_persp_correct_band", (0,))[0] == -(-oh // 64), sorted(prof)


def test_cpp_write_sweep_equals_reference(tmp_path):
    """B200CylinderBlender::write_sweep (openpano_b200/host/pano_host_io.hh) next to the reference's read_img,
    CylinderWarper, blenders, perspective_correction, crop and write_rgb on PNG and PPM files, file bytes; and the
    corner points b200_correction_points gives next to those the reference's perspective_correction hands to
    getPerspectiveTransform (oracle/_ref/cyl_sweep_test)."""
    import os
    import subprocess
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    binary = root / "oracle" / "_ref" / "cyl_sweep_test"
    if not binary.exists():
        pytest.skip("oracle/_ref/cyl_sweep_test not built (needs the reference sources at build time)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{root / 'oracle' / '_ref'}:{root / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(binary), str(tmp_path)], capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "CYL SWEEP TEST OK" in out.stdout
    assert out.stdout.count("file bytes identical") == 4 * 2 * 2 * 2 * 3
    assert out.stdout.count("correction points identical") == 50


def _strided(x):
    """x's pixels in an array that is not C-contiguous: the first channels of a wider pixel, or every other row."""
    if x.ndim == 3 and x.dtype == np.uint8:
        wide = np.zeros(x.shape[:2] + (x.shape[2] + 1,), x.dtype)
        wide[..., :x.shape[2]] = x
        v = wide[..., :x.shape[2]]
    else:
        tall = np.zeros((2 * x.shape[0],) + x.shape[1:], x.dtype)
        tall[::2] = x
        v = tall[::2]
    assert not v.flags.c_contiguous and np.array_equal(v, x)
    return v


@pytest.mark.parametrize("fmt", ["rgb", "grey", "f32"])
def test_non_contiguous_sources(engine, fmt):
    """numpy sources that are views, not C-contiguous arrays: both sweeps read copies of them that live until the
    sweep has run, and give the bytes of the contiguous sources."""
    from openpano_b200.stitcher import mosaic_rgb8_sweep
    rgb, items, geom = _case(n=5)
    srcs = [_layout(x, fmt) for x in rgb]
    views = [_strided(x) for x in srcs]
    fmts = None if fmt == "f32" else [fmt] * 5
    inv = pu.inv_cases(max(it[2] for it in items), max(it[3] for it in items), seed=2)["keystone"]
    for rows in (1, 40):
        want = _sweep(engine, items, geom, inv, 0, srcs, [fmt] * 5, rows, 0)[:2]
        got = _sweep(engine, items, geom, inv, 0, views, [fmt] * 5, rows, 0)[:2]
        assert np.array_equal(got[0], want[0]) and gu.same_bits(got[1], want[1]), rows
    # the plain sweep, over the sources' own shapes
    imgs, org = synth.make_stack(5, 160, 120, 50, 19)
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    srcs = [_layout(x, fmt) for x in pix]
    views = [_strided(x) for x in srcs]
    items, geom = synth.translation_blend_setup(org, 160, 120)
    for rows in (1, 40):
        want = mosaic_rgb8_sweep(engine, items, geom, 0, srcs, rows, 0, fmt=fmts)
        got = mosaic_rgb8_sweep(engine, items, geom, 0, views, rows, 0, fmt=fmts)
        assert np.array_equal(got[0], want[0]) and gu.same_bits(got[1], want[1]), rows
