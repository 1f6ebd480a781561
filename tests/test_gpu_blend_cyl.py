"""GPU: cylinder mode's blend from the unwarped sources (pano_blend_stream_create_cyl).  The mosaic must have the raw
bits of warping first — pano_cyl_warp_batch[_rgb8]_dev, then pano_blend_dev over the warped images — for every
source kind and PANO_PIX_* format, every window partition, both blenders and the h_factor values the h-factor
search tries; at config 1's shape it must equal the oracle's warp + blend as well.  Also the misuse rules, the
memory bound, and the C++ drop-in (B200CylinderBlender) next to the reference's own CylinderWarper and blenders."""
import ctypes as C
import math
import os
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from openpano_b200.capi import (PIX_FORMATS, SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_DEV, SRC_RGB8_HOST, Engine,
                                PanoError)
from tests import golden_util as gu
from tests.pix_util import to_planar, to_rgba

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "cyl_blend_test"
MB = 1 << 20


def _layout(rgb, fmt):
    """8-bit pixels in a PANO_PIX_* layout, or read_img's f32 image for fmt "f32"."""
    if fmt == "grey":
        return np.ascontiguousarray(rgb[..., 1])
    if fmt == "rgb":
        return rgb
    if fmt == "rgba":
        return to_rgba(rgb, alpha_seed=5)
    if fmt == "planar":
        return to_planar(rgb)
    assert fmt == "f32"
    return (rgb.astype(np.float64) / 255.0).astype(np.float32)


def _code(fmt):
    return 3 if fmt == "f32" else PIX_FORMATS[fmt]


def _case(n=6, w=240, h=180, step=70, seed=11, h_factor=1.0, params=None):
    """n 8-bit sources and the items / geometry of their warped images on a flat canvas: a slight rotation and
    sub-pixel shifts, so that blend taps fall between warped pixels."""
    imgs, org = synth.make_stack(n, w, h, step, seed)
    rgb = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    ow, oh, _, _ = Engine.cyl_warp_shape(w, h, h_factor, params)
    homos, boxes = [], []
    for k, (x, y) in enumerate(org):
        th = 0.004 * (k - n / 2)
        H = np.array([[math.cos(th), -math.sin(th), x + 0.37 * k], [math.sin(th), math.cos(th), 0.61 * k],
                      [0.0, 0.0, 1.0]])
        corners = np.array([[sx * ow / 2, sy * oh / 2, 1.0] for sx in (-1, 1) for sy in (-1, 1)]) @ H.T
        homos.append(list(np.linalg.inv(H).ravel()))
        boxes.append((corners[:, 0].min(), corners[:, 1].min(), corners[:, 0].max(), corners[:, 1].max()))
    mx, my = math.floor(min(b[0] for b in boxes)), math.floor(min(b[1] for b in boxes))
    items = [(int(b[0] - mx), int(b[1] - my), int(b[2] - mx), int(b[3] - my), hi) for b, hi in zip(boxes, homos)]
    geom = dict(projection=0, res_x=1.0, res_y=1.0, proj_min_x=float(mx), proj_min_y=float(my))
    return rgb, items, geom


def _warp_then_blend(eng, srcs, codes, items, geom, bands, h_factor, params=None):
    """The mosaic of warping first: the batched warp of the sources on the device, then blend_dev over the warped
    images.  codes: one PANO_PIX_* code per source, or 3 for all-f32 sources."""
    params = params or default_params()
    f32 = srcs[0].dtype == np.float32
    shapes = [s.shape[1:] if c == PIX_FORMATS["planar"] else s.shape[:2] for s, c in zip(srcs, codes)]
    ws = [Engine.cyl_warp_shape(w, h, h_factor, params) for h, w in shapes]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    d_src = [eng.dev_alloc(s.nbytes) for s in srcs]
    d_warp = [eng.dev_alloc(oh * ow * 12) for ow, oh, _, _ in ws]
    d_out = eng.dev_alloc(tw * th * 12)
    try:
        for d, s in zip(d_src, srcs):
            eng.dev_upload(d, s)
        if f32:
            eng.cyl_warp_batch_dev(d_src, shapes, d_warp, None, h_factor, params)
        else:
            eng.cyl_warp_batch_rgb8_dev(d_src, codes, shapes, d_warp, None, h_factor, params)
        eng.blend_dev(d_warp, [(oh, ow) for ow, oh, _, _ in ws], items, geom, d_out, tw, th, bands, params)
        out = np.empty((th, tw, 3), np.float32)
        eng.dev_download(out, d_out)
    finally:
        for d in d_src + d_warp + [d_out]:
            eng.dev_free(d)
    return out


def _stream(eng, srcs, fmts, items, geom, bands, h_factor, windows, params=None):
    """The cylinder stream fed pageable host windows: windows is a list of sizes, fmts one format per source."""
    shapes = [s.shape[1:] if f == "planar" else s.shape[:2] for s, f in zip(srcs, fmts)]
    s = eng.blend_stream_cyl(shapes, items, geom, h_factor, bands, params)
    try:
        k = 0
        for q in windows:
            s.add(srcs[k:k + q], fmt=None if fmts[k] == "f32" else fmts[k])
            k += q
        assert k == len(srcs)
        return s.finish()
    finally:
        s.close()


def _windows(name, n):
    return {"1": [1] * n, "3": [3] * (n // 3) + ([n % 3] if n % 3 else []), "n": [n]}[name]


@pytest.mark.parametrize("fmt", ["grey", "rgb", "rgba", "planar", "f32"])
@pytest.mark.parametrize("bands", [0, 5])
def test_every_format_and_window_equals_warp_then_blend(engine, fmt, bands):
    rgb, items, geom = _case()
    srcs = [_layout(x, fmt) for x in rgb]
    want = _warp_then_blend(engine, srcs, [_code(fmt)] * len(srcs), items, geom, bands, 1.0)
    assert (want[..., 0] == -1).any() and (want[..., 0] >= 0).mean() > 0.5
    for name in ("1", "3", "n"):
        got = _stream(engine, srcs, [fmt] * len(srcs), items, geom, bands, 1.0, _windows(name, len(srcs)))
        assert gu.same_bits(got, want), (fmt, bands, name)


@pytest.mark.parametrize("bands", [0, 2])
def test_mixed_formats_in_one_stream(engine, bands):
    """One window per format; the reference warps the whole mixed batch in one launch."""
    rgb, items, geom = _case(n=8)
    fmts = ["rgb", "rgb", "grey", "rgba", "rgba", "planar", "grey", "rgb"]
    srcs = [_layout(x, f) for x, f in zip(rgb, fmts)]
    want = _warp_then_blend(engine, srcs, [_code(f) for f in fmts], items, geom, bands, 1.0)
    assert gu.same_bits(_stream(engine, srcs, fmts, items, geom, bands, 1.0, [2, 1, 2, 1, 1, 1]), want)


@pytest.mark.parametrize("lazy,ordered", [(1, 0), (1, 1), (0, 0), (0, 1)])
@pytest.mark.parametrize("h_factor", [1.0, 0.8, 1.2])
def test_linear_flags_and_h_factor(engine, lazy, ordered, h_factor):
    p = default_params(lazy_read=lazy, ordered_input=ordered)
    rgb, items, geom = _case(n=7, h_factor=h_factor, params=p)
    want = _warp_then_blend(engine, rgb, [3] * 7, items, geom, 0, h_factor, p)
    for name in ("1", "3", "n"):
        got = _stream(engine, rgb, ["rgb"] * 7, items, geom, 0, h_factor, _windows(name, 7), p)
        assert gu.same_bits(got, want), name


@pytest.mark.parametrize("bands", [1, 2, 5])
@pytest.mark.parametrize("h_factor", [1.0, 0.8, 1.2])
def test_multiband_bands_and_h_factor(engine, bands, h_factor):
    rgb, items, geom = _case(n=7, h_factor=h_factor)
    want = _warp_then_blend(engine, rgb, [3] * 7, items, geom, bands, h_factor)
    for name in ("1", "3", "n"):
        got = _stream(engine, rgb, ["rgb"] * 7, items, geom, bands, h_factor, _windows(name, 7))
        assert gu.same_bits(got, want), name


@pytest.mark.parametrize("bands", [0, 3])
def test_all_source_kinds(engine, bands):
    """Device and host sources, f32 and 8-bit, pageable and pinned host buffers, in one stream and one kind per
    stream."""
    rgb, items, geom = _case(n=8)
    f32 = [_layout(x, "f32") for x in rgb]
    want = _warp_then_blend(engine, rgb, [3] * 8, items, geom, bands, 1.0)
    assert gu.same_bits(_warp_then_blend(engine, f32, [3] * 8, items, geom, bands, 1.0), want)
    shapes = [x.shape[:2] for x in rgb]
    d_f32 = [engine.dev_alloc(x.nbytes) for x in f32]
    d_pix = [engine.dev_alloc(x.nbytes) for x in rgb]
    h_f32 = [Engine.host_alloc(x.nbytes) for x in f32]
    h_pix = [Engine.host_alloc(x.nbytes) for x in rgb]
    try:
        for d, h, x in zip(d_f32 + d_pix, h_f32 + h_pix, f32 + rgb):
            engine.dev_upload(d, x)
            C.memmove(h, x.ctypes.data, x.nbytes)
        s = engine.blend_stream_cyl(shapes, items, geom, 1.0, bands)
        try:
            s.add(d_f32[0:2], SRC_F32_DEV)
            s.add(h_pix[2:3], SRC_RGB8_HOST)             # pinned
            s.add(f32[3:4])                               # pageable f32
            s.add(d_pix[4:6], SRC_RGB8_DEV)
            s.add(h_f32[6:7], SRC_F32_HOST)              # pinned
            s.add(rgb[7:8])                               # pageable u8
            got = s.finish()
        finally:
            s.close()
        assert gu.same_bits(got, want)
        for kind, ptrs in ((SRC_F32_DEV, d_f32), (SRC_F32_HOST, h_f32), (SRC_RGB8_DEV, d_pix), (SRC_RGB8_HOST, h_pix)):
            for win in (1, 3, 8):
                s = engine.blend_stream_cyl(shapes, items, geom, 1.0, bands)
                d_out = engine.dev_alloc(want.nbytes)
                try:
                    for k in range(0, 8, win):
                        s.add(ptrs[k:k + win], kind)
                    s.finish_dev(d_out)
                    got = np.empty_like(want)
                    engine.dev_download(got, d_out)
                finally:
                    s.close()
                    engine.dev_free(d_out)
                assert gu.same_bits(got, want), (kind, win)
    finally:
        for d in d_f32 + d_pix:
            engine.dev_free(d)
        for h in h_f32 + h_pix:
            Engine.host_free(h)


@pytest.mark.parametrize("shape", [(4, 4), (3, 5), (3, 61), (60, 4), (5, 200)])
@pytest.mark.parametrize("bands", [0, 2])
def test_small_and_thin_shapes(engine, shape, bands):
    """Sources whose warp is 2 pixels wide or tall (4×4 -> 2×3, 3×5 -> 3×2) and thin strips."""
    h, w = shape
    ow, oh, _, _ = Engine.cyl_warp_shape(w, h)
    assert min(ow, oh) >= 2
    rng = np.random.RandomState(h * 1000 + w)
    rgb = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for _ in range(3)]
    org = [(0, 0), (1, 0), (1, 1)]
    items, geom = synth.translation_blend_setup(org, ow, oh)
    for fmt in ("rgb", "grey", "rgba", "planar", "f32"):
        srcs = [_layout(x, fmt) for x in rgb]
        want = _warp_then_blend(engine, srcs, [_code(fmt)] * 3, items, geom, bands, 1.0)
        for win in ([1, 1, 1], [3]):
            assert gu.same_bits(_stream(engine, srcs, [fmt] * 3, items, geom, bands, 1.0, win), want), (fmt, win)


def test_config1_against_the_oracle(engine, orc):
    """BASELINE config 1 (CMU0, cylinder mode) at its shape: the stream on the 8-bit sources equals the oracle's
    CylinderWarper::warp of every read_img image followed by LinearBlender over the warped images, as
    test_config1_cmu0_cylinder_hot_path checks the warp-then-blend path."""
    from tests.checker import get_checker
    omt = get_checker("orc_mt")
    views, org = synth.config_stack("cmu0_8x600x400")
    pix = [(v * 255.0 + 0.5).astype(np.uint8) for v in views]
    imgs = [orc.read_img_rgb8(x) for x in pix]
    n, (h, w) = len(imgs), imgs[0].shape[:2]
    params = default_params(ordered_input=1)
    ow, oh, _, _ = engine.cyl_warp_shape(w, h, 1.0, params)
    assert (ow, oh) == orc.cyl_warp_shape(w, h, 1.0, params)[:2]
    warped = [orc.cyl_warp(im, np.zeros((0, 2)), 1.0, params)[0] for im in imgs]
    items, geom = synth.translation_blend_setup(org, ow, oh)
    want = omt.blend(warped, items, geom, 0, params)
    for win in ([1] * n, [3, 3, 2], [n]):
        assert gu.same_bits(_stream(engine, pix, ["rgb"] * n, items, geom, 0, 1.0, win, params), want), win


def test_profile_names(engine):
    """Each tap source's kernels under their own name, one launch per window."""
    rgb, items, geom = _case(n=4)
    for fmt, suffix in (("f32", "_cyl"), ("rgb", "_cyl_rgb8"), ("grey", "_cyl_rgb8"), ("rgba", "_cyl_pix8"),
                        ("planar", "_cyl_pix8")):
        srcs = [_layout(x, fmt) for x in rgb]
        for bands, kernel in ((0, "k_linear_accumulate"), (2, "k_mb_first_level")):
            engine.profile(True)
            engine.profile_reset()
            try:
                _stream(engine, srcs, [fmt] * 4, items, geom, bands, 1.0, [1, 3])
                prof = engine.profile_read()
            finally:
                engine.profile(False)
            assert prof.get(kernel + suffix, (0,))[0] == 2, (fmt, bands, sorted(prof))


def test_misuse_is_invalid_and_sticky(engine):
    from openpano_b200.capi import LIB
    rgb, items, geom = _case(n=4)
    h, w = rgb[0].shape[:2]
    p = default_params()
    ow, oh, _, _ = Engine.cyl_warp_shape(w, h, 1.0, p)
    shapes = [(oh, ow)] * 4
    arr, g = engine._blend_args([None] * 4, shapes, items, geom)
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    sw, sh = (C.c_int * 4)(*[w] * 4), (C.c_int * 4)(*[h] * 4)
    hnd = C.c_void_p()
    create = LIB.pano_blend_stream_create_cyl
    assert create(engine._h, 4, arr, sw, sh, 1.0, C.byref(g), 0, C.byref(p), tw, th, C.byref(hnd)) == 0
    LIB.pano_blend_stream_free(hnd)
    # a warped shape other than pano_cyl_warp_shape's, a source under 2×2, a warp under 2×2, null lists
    for dw, dh in [(1, 0), (0, -1)]:
        bad, _ = engine._blend_args([None] * 4, [(oh + dh, ow + dw)] + shapes[1:], items, geom)
        assert create(engine._h, 4, bad, sw, sh, 1.0, C.byref(g), 0, C.byref(p), tw, th, C.byref(hnd)) == -2, (dw, dh)
        assert "warps to" in LIB.pano_last_error(engine._h).decode()
    one = (C.c_int * 4)(1, w, w, w)
    assert create(engine._h, 4, arr, one, sh, 1.0, C.byref(g), 0, C.byref(p), tw, th, C.byref(hnd)) == -2
    assert create(engine._h, 4, arr, None, sh, 1.0, C.byref(g), 0, C.byref(p), tw, th, C.byref(hnd)) == -2
    assert create(engine._h, 4, arr, sw, sh, 1.0, C.byref(g), 0, C.byref(p), tw + 1, th, C.byref(hnd)) == -2
    assert create(engine._h, 4, arr, sw, sh, 1.0, C.byref(g), 0, C.byref(p), tw, th, None) == -2
    assert create(None, 4, arr, sw, sh, 1.0, C.byref(g), 0, C.byref(p), tw, th, C.byref(hnd)) == -2
    with pytest.raises(PanoError) as ei:
        engine.blend_stream_cyl([(2, 2)] * 4, items, geom, 1.0)        # its warp is 1×0
    assert ei.value.code == -2
    with pytest.raises(PanoError) as ei:
        engine.blend_stream_cyl([(2, 40)] * 4, items, geom, 1.0)       # 2×N: its warp is 1 row tall
    assert ei.value.code == -2
    # adds in the unwarped shape only; every failure sticks
    s = engine.blend_stream_cyl([(h, w)] * 4, items, geom, 1.0)
    try:
        with pytest.raises(PanoError):
            s.add([np.zeros((oh, ow, 3), np.uint8)])                  # the warped shape is not the source's
        with pytest.raises(PanoError):
            s.add(rgb[0:1])
    finally:
        s.close()
    out = np.empty((th, tw, 3), np.float32)
    fp = C.POINTER(C.c_float)
    srcs = (C.c_void_p * 4)(*[x.ctypes.data for x in rgb])
    add = LIB.pano_blend_stream_add
    for name, call in {
        "out of order": lambda hd: add(hd, 1, 1, srcs, SRC_RGB8_HOST, 3),
        "unknown format": lambda hd: add(hd, 0, 1, srcs, SRC_RGB8_HOST, 2),
        "finish early": lambda hd: (add(hd, 0, 2, srcs, SRC_RGB8_HOST, 3),
                                    LIB.pano_blend_stream_finish(hd, out.ctypes.data_as(fp)))[1],
    }.items():
        assert create(engine._h, 4, arr, sw, sh, 1.0, C.byref(g), 0, C.byref(p), tw, th, C.byref(hnd)) == 0
        try:
            assert call(hnd) == -2, name
            assert add(hnd, 0, 4, srcs, SRC_RGB8_HOST, 3) == -2, f"{name}: not sticky"
            assert LIB.pano_blend_stream_finish(hnd, out.ctypes.data_as(fp)) == -2, f"{name}: not sticky"
        finally:
            LIB.pano_blend_stream_free(hnd)
    # the context is still usable
    want = _warp_then_blend(engine, rgb, [3] * 4, items, geom, 0, 1.0)
    assert gu.same_bits(_stream(engine, rgb, ["rgb"] * 4, items, geom, 0, 1.0, [2, 2]), want)


def _canvas_state(items, tw, th, bands):
    """The stream's canvas state as include/pano_b200.h states it (finish()'s output included)."""
    if bands == 0:
        return 16 * tw * th
    roi = sum(-(-(x1 - x0 + 1) // 32) * 32 * (y1 - y0 + 1) for x0, y0, x1, y1, _ in items)
    return 33 * roi + tw * th + 12 * tw * th


@pytest.mark.parametrize("bands", [0, 5])
def test_memory_bound(monkeypatch, bands):
    """13 × 1500×1112 8-bit sources, two per window: the pool's high-water mark stays within the canvas state, two
    windows of sources, the column tables and 64 MB, and below warping first (8-bit sources and every warped f32
    image on the device, then pano_blend_dev).  Both give the same bits."""
    monkeypatch.setenv("PANO_CACHE_MB", "0")
    n, w, h = 13, 1500, 1112
    org = [(k * 500, 0) for k in range(n)]
    rng = np.random.RandomState(7)
    pix = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for _ in range(n)]
    eng = Engine(0)
    try:
        ow, oh, _, _ = eng.cyl_warp_shape(w, h)
        items, geom = synth.translation_blend_setup(org, ow, oh)
        eng.trim()
        eng.sync()
        eng.mem_high_water(reset=True)
        s = eng.blend_stream_cyl([(h, w)] * n, items, geom, 1.0, bands)
        try:
            for k in range(0, n, 2):
                s.add(pix[k:k + 2])
            got = s.finish()
        finally:
            s.close()
        eng.sync()
        stream_mark = eng.mem_high_water(reset=True)
        th, tw = got.shape[:2]
        bound = _canvas_state(items, tw, th, bands) + 2 * 2 * pix[0].nbytes + 16 * ow * n + 64 * MB
        assert stream_mark <= bound, (stream_mark / MB, bound / MB)
        want = _warp_then_blend(eng, pix, [3] * n, items, geom, bands, 1.0)
        eng.sync()
        warp_mark = eng.mem_high_water()
        assert gu.same_bits(got, want)
        assert stream_mark < warp_mark, (stream_mark / MB, warp_mark / MB)
        print(f"bands={bands}: stream {stream_mark / MB:.0f} MB (bound {bound / MB:.0f} MB), "
              f"warp then blend {warp_mark / MB:.0f} MB")
    finally:
        eng.close()


def test_cpp_cylinder_blender_equals_reference(tmp_path):
    """B200CylinderBlender (openpano_b200/host/pano_host.hh) on the unwarped images next to the reference's
    CylinderWarper + LinearBlender (LAZY_READ 1 and 0, ORDERED_INPUT 1 and 0) and MultiBandBlender over the warped
    ones, compiled against the reference's headers (oracle/_ref/cyl_blend_test)."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/cyl_blend_test not built (needs the reference sources at build time)")
    h_factor = 0.9
    rgb, items, geom = _case(n=5, w=200, h=150, step=60, seed=53, h_factor=h_factor)
    imgs = [_layout(x, "f32") for x in rgb]
    path = tmp_path / "stack.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<3i", len(imgs), 200, 150))
        for im in imgs:
            f.write(np.ascontiguousarray(im, np.float32).tobytes())
        f.write(struct.pack("<d", h_factor))
        for it in items:
            f.write(struct.pack("<4i", *it[:4]))
            f.write(struct.pack("<9d", *it[4]))
        f.write(struct.pack("<3d", geom["res_x"], geom["proj_min_x"], geom["proj_min_y"]))
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(path)], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "CYL BLEND TEST OK" in out.stdout
    assert out.stdout.count("identical") == 15
