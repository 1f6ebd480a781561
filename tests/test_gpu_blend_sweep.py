"""GPU: the blend sweep (pano_blend_sweep_*).  Its bytes must equal the whole-canvas path's (blend + crop +
write_rgb's conversion) and mosaic_rgb8_strips', for every source kind and PANO_PIX_* format (mixed in one sweep),
linear and multiband, all projections, crop on and off, every output layout, keep budgets from none to unlimited and
strip heights from 1 row to more than the canvas; its hand-overs must be the plan's; its read sets those of row
streams; misuse must be sticky; and its device memory must stay within the header's bound."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200.capi import (PIX_FORMATS, SIZE_MAX, SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_DEV, SRC_RGB8_HOST, Engine,
                                blend_sweep_plan, pix_format)
from openpano_b200.stitcher import mosaic_rgb8_strips, mosaic_rgb8_sweep
from tests import golden_util as gu
from tests.test_gpu_blend_strips import _as_format, _canvas, _gap_stack, _pix, _stack, _strip_state
from tests.test_gpu_match_warp_blend import _perspective_items

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "blend_sweep_test"
MB = 1 << 20
FORMATS = ["grey", "rgb", "rgba", "planar"]


def _mixed(pix):
    """Image k in format FORMATS[k % 4]: (pixels, fmt names, PANO_PIX_* codes)."""
    fmts = [FORMATS[k % 4] for k in range(len(pix))]
    return [_as_format(x, f) for x, f in zip(pix, fmts)], fmts, [PIX_FORMATS[f] for f in fmts]


def _whole(engine, pix, fmts, items, geom, bands, crop, out):
    f32 = [engine.read_img_rgb8(x, fmt=f) for x, f in zip(pix, fmts)]
    return engine.crop_write_pix8(engine.blend(f32, items, geom, bands), crop, out)


def _keeps(shapes, items, geom, bands, rows, nbytes):
    live = blend_sweep_plan(shapes, items, geom, bands, rows, nbytes, SIZE_MAX)["retained_high"]
    return [0, max(nbytes), live, SIZE_MAX]


def _check_sweep(engine, items, geom, bands, srcs, rows, keep, want_rect, want, crop, out, **kw):
    st = {}
    rect, got = mosaic_rgb8_sweep(engine, items, geom, bands, srcs, rows, keep, out, crop, stats=st, **kw)
    assert (rect is None) == (not crop)
    if crop:
        assert np.array_equal(rect, want_rect), (rows, keep)
    assert gu.same_bits(got, want), (rows, keep, crop, out)
    return st


@pytest.mark.parametrize("projection", [0, 1, 2])
@pytest.mark.parametrize("bands", [0, 1, 2, 5])
def test_sweep_equals_whole_canvas(engine, projection, bands):
    """Pageable host sources in all four formats in one sweep; strips of 1, 37, the canvas and more; every budget."""
    imgs, org = synth.make_stack(5, 300, 200, 100, 7)
    items, geom = _perspective_items(org, 5, projection)
    pix, fmts, codes = _mixed(_pix(imgs))
    shapes = [pix_format(x, f)[1:] for x, f in zip(pix, fmts)]
    nbytes = [x.nbytes for x in pix]
    ow, oh = _canvas(items)
    for crop, out in ((True, "rgb"), (False, "rgba"), (True, "planar")):
        want_rect, want = _whole(engine, pix, fmts, items, geom, bands, crop, out)
        for rows in ((1, 37, oh, oh + 3) if crop and out == "rgb" else (37,)):
            for keep in _keeps(shapes, items, geom, bands, rows, nbytes):
                st = _check_sweep(engine, items, geom, bands, pix, rows, keep, want_rect, want, crop, out, fmt=fmts)
                pl = blend_sweep_plan(shapes, items, geom, bands, rows, nbytes, keep)
                assert (st["uploads"], st["upload_bytes"], st["retained_high"]) == \
                    (pl["n_uploads"], pl["upload_bytes"], pl["retained_high"]), (rows, keep)


@pytest.mark.parametrize("bands", [0, 5])
@pytest.mark.parametrize("out", ["rgb", "rgba", "planar"])
def test_sweep_equals_strips(engine, bands, out):
    """One format per sweep, as mosaic_rgb8_strips takes: both give the same bytes, the sweep with fewer uploads."""
    imgs, items, geom = _stack(7)
    items, imgs = items[:3] + items[4:], imgs[:3] + imgs[4:]
    pix = _pix(imgs)
    for rows in (1, 256, 40):
        want_rect, want = mosaic_rgb8_strips(engine, items, geom, bands, pix, rows, 1, out, True)
        nb = [x.nbytes for x in pix]
        none = _check_sweep(engine, items, geom, bands, pix, rows, 0, want_rect, want, True, out)
        once = _check_sweep(engine, items, geom, bands, pix, rows, SIZE_MAX, want_rect, want, True, out)
        assert once["upload_bytes"] == sum(nb)
        assert none["upload_bytes"] >= once["upload_bytes"]


def _pointer_sources(engine, kind, srcs):
    host = kind in (SRC_F32_HOST, SRC_RGB8_HOST)
    ptrs = [Engine.host_alloc(x.nbytes) if host else engine.dev_alloc(x.nbytes) for x in srcs]
    for q, x in zip(ptrs, srcs):
        if host:
            C.memmove(q, x.ctypes.data, x.nbytes)
        else:
            engine.dev_upload(q, x)
    return ptrs, host


@pytest.mark.parametrize("kind", ["rgb8_host_pinned", "rgb8_dev", "f32_host_pinned", "f32_dev", "f32_pageable"])
@pytest.mark.parametrize("bands", [0, 2])
def test_sweep_source_kinds(engine, kind, bands):
    imgs, items, geom = _gap_stack()
    pix, fmts, codes = _mixed(_pix(imgs))
    f32 = [engine.read_img_rgb8(x, fmt=f) for x, f in zip(pix, fmts)]
    shapes = [x.shape[:2] for x in f32]
    want_rect, want = engine.crop_write_pix8(engine.blend(f32, items, geom, bands), True, "planar")
    u8 = kind.startswith("rgb8")
    srcs = pix if u8 else f32
    nbytes = [x.nbytes for x in srcs]
    for rows in (1, 33):
        for keep in _keeps(shapes, items, geom, bands, rows, nbytes):
            if kind == "f32_pageable":
                st = _check_sweep(engine, items, geom, bands, f32, rows, keep, want_rect, want, True, "planar")
            else:
                code = {"rgb8_host_pinned": SRC_RGB8_HOST, "rgb8_dev": SRC_RGB8_DEV, "f32_host_pinned": SRC_F32_HOST,
                        "f32_dev": SRC_F32_DEV}[kind]
                ptrs, host = _pointer_sources(engine, code, srcs)
                try:
                    st = _check_sweep(engine, items, geom, bands, ptrs, rows, keep, want_rect, want, True, "planar",
                                      kind=code, formats=codes if u8 else None, shapes=shapes)
                finally:
                    for q in ptrs:
                        Engine.host_free(q) if host else engine.dev_free(q)
            pl = blend_sweep_plan(shapes, items, geom, bands, rows, nbytes, keep)
            assert (st["uploads"], st["upload_bytes"], st["retained_high"]) == \
                (pl["n_uploads"], pl["upload_bytes"], pl["retained_high"])


@pytest.mark.parametrize("bands", [0, 1, 5])
def test_plan_reads_equal_stream_needs(engine, bands):
    imgs, items, geom = _gap_stack()
    shapes = [x.shape[:2] for x in imgs]
    ow, oh = _canvas(items)
    for rows in (1, 29, oh):
        pl = blend_sweep_plan(shapes, items, geom, bands, rows, [1] * len(items), 0)
        for s, r0 in enumerate(range(0, oh, rows)):
            bs = engine.blend_stream_rows(shapes, items, geom, r0, min(oh, r0 + rows), bands)
            try:
                assert np.array_equal(bs.needs(), pl["reads"][s]), (rows, s)
            finally:
                bs.close()


def test_gap_strips_and_wide_canvas(engine):
    """Strips no image reaches come out as -1 (white once converted); a canvas over 40,000 columns crops through
    the crop scan's global-memory line kernel."""
    imgs, items, geom = _gap_stack()
    pix = _pix(imgs)
    for bands in (0, 2):
        want_rect, want = _whole(engine, pix, [None] * len(pix), items, geom, bands, False, "rgb")
        assert (want == 255).all(axis=2).all(axis=1).any()
        _check_sweep(engine, items, geom, bands, pix, 16, SIZE_MAX, None, want, False, "rgb")
    n, w, h = 40, 1200, 90
    imgs, org = synth.make_stack(n, w, h, 1000, 61)
    org = [(x, y + (k * 7) % 23) for k, (x, y) in enumerate(org)]
    items, geom = synth.translation_blend_setup(org, w, h)
    assert _canvas(items)[0] > 40000
    pix = _pix(imgs)
    want_rect, want = mosaic_rgb8_strips(engine, items, geom, 0, pix, 32, 4)
    assert 0 < want_rect[3] < _canvas(items)[1]
    _check_sweep(engine, items, geom, 0, pix, 32, SIZE_MAX, want_rect, want, True, "rgb")


def test_misuse_is_invalid_and_sticky(engine):
    from openpano_b200.capi import PanoError
    imgs, items, geom = _gap_stack()
    pix = _pix(imgs)
    n = len(pix)
    shapes = [x.shape[:2] for x in pix]
    ptrs = [x.ctypes.data for x in pix]
    d_out = engine.dev_alloc(_canvas(items)[0] * _canvas(items)[1] * 4)
    try:
        def sweep():
            return engine.blend_sweep(shapes, items, geom, 40, SIZE_MAX, 0)

        def expect_sticky(sw, call):
            with pytest.raises(PanoError) as ei:
                call()
            assert ei.value.code == -2
            with pytest.raises(PanoError) as ei:                 # sticky: the next call fails the same way
                sw.strip([0] * n, [3] * n, SRC_RGB8_HOST)
            assert ei.value.code == -2

        # a source missing where want is set; an extra source
        for extra in (False, True):
            sw = sweep()
            try:
                st, want = sw.next()
                assert st == 0 and want.any() and not want.all()
                k = int(np.argmin(want)) if extra else int(np.argmax(want))
                bad = [q if (w != (j == k)) else 0 for j, (q, w) in enumerate(zip(ptrs, want))]
                if extra:
                    bad[k] = ptrs[k]
                expect_sticky(sw, lambda: sw.strip(bad, [3] * n, SRC_RGB8_HOST))
            finally:
                sw.close()
        # finish before the last strip, a strip after the last, a second finish
        sw = sweep()
        try:
            expect_sticky(sw, lambda: sw.finish_dev("rgb", d_out))
        finally:
            sw.close()
        sw = sweep()
        try:
            while True:
                st, want = sw.next()
                if st < 0:
                    break
                sw.strip([q if w else 0 for q, w in zip(ptrs, want)], [3] * n, SRC_RGB8_HOST)
            assert sw.next()[0] == -1
            sw.finish_dev("rgb", d_out)
            with pytest.raises(PanoError) as ei:
                sw.finish_dev("rgb", d_out)
            assert ei.value.code == -2
        finally:
            sw.close()
        sw = sweep()
        try:
            for _ in range(20):
                st, want = sw.next()
                if st < 0:
                    break
                sw.strip([q if w else 0 for q, w in zip(ptrs, want)], [3] * n, SRC_RGB8_HOST)
            expect_sticky(sw, lambda: sw.strip([0] * n, [3] * n, SRC_RGB8_HOST))
        finally:
            sw.close()
    finally:
        engine.dev_free(d_out)
    # the context is still usable
    want_rect, want = _whole(engine, pix, [None] * n, items, geom, 0, True, "rgb")
    _check_sweep(engine, items, geom, 0, pix, 40, SIZE_MAX, want_rect, want, True, "rgb")


@pytest.mark.parametrize("bands", [0, 5])
def test_pool_bound(monkeypatch, bands):
    """Strips of 512 rows of a 40-image mosaic, every budget: the pool's high-water mark stays within the header's
    device-memory bound."""
    monkeypatch.setenv("PANO_CACHE_MB", "0")
    w, h, n = 2000, 1500, 40
    base = np.random.RandomState(4).randint(0, 256, (h + 4 * 750, w + 7 * 1000, 3), dtype=np.uint8)
    org = [(c * 1000, r * 750) for r in range(5) for c in range(8)]
    pix = [np.ascontiguousarray(base[y:y + h, x:x + w]) for x, y in org]
    items, geom = synth.translation_blend_setup(org, w, h)
    shapes = [x.shape[:2] for x in pix]
    nbytes = [x.nbytes for x in pix]
    tw, th = _canvas(items)
    rows = 512
    eng = Engine(0)
    try:
        want_rect, want = mosaic_rgb8_strips(eng, items, geom, bands, pix, rows, 2, "rgb", True)
        state = max(_strip_state(items, tw, r0, min(th, r0 + rows), th, bands) for r0 in range(0, th, rows))
        for keep in _keeps(shapes, items, geom, bands, rows, nbytes):
            pl = blend_sweep_plan(shapes, items, geom, bands, rows, nbytes, keep)
            reads = [sum(b for b, r in zip(nbytes, rd) if r) for rd in pl["reads"]]
            bound = (state + 12 * tw * rows + 6 * tw * th + 2 * max(nbytes) + pl["retained_high"] + max(reads)
                     + 64 * MB)
            eng.trim()
            eng.sync()
            eng.mem_high_water(reset=True)
            _check_sweep(eng, items, geom, bands, pix, rows, keep, want_rect, want, True, "rgb")
            eng.sync()
            mark = eng.mem_high_water()
            assert mark <= bound, (keep, mark / MB, bound / MB)
            print(f"bands={bands} keep={min(keep, 1 << 50) / MB:.0f} MB: pool {mark / MB:.0f} MB "
                  f"(bound {bound / MB:.0f} MB), uploaded {pl['upload_bytes'] / MB:.0f} MB")
    finally:
        eng.close()


def test_cpp_write_sweep_equals_reference(tmp_path):
    """B200PixelBlender::write_sweep (openpano_b200/host/pano_host_io.hh) next to the reference's blenders, crop() and
    write_rgb() on PNG, PPM and PGM files (oracle/_ref/blend_sweep_test)."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/blend_sweep_test not built (needs the reference sources at build time)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(tmp_path)], capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "BLEND SWEEP TEST OK" in out.stdout
    assert out.stdout.count("identical") > 0
