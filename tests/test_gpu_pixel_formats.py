"""GPU: the 8-bit entry points in the layouts of the reference's decoders and encoders — lodepng's RGBA
(PANO_PIX_RGBA, read_png / write_png) and CImg's planes (PANO_PIX_RGB_PLANAR, read_img / write_rgb).  Every
result must have the raw bits of the interleaved path (PANO_PIX_RGB) on the same colour pixels, whatever the
fourth byte holds; grey-valued RGBA is divided by 255 unlike PANO_PIX_GREY; the output conversion matches the
plain-C restatement of write_png's and write_rgb's buffers (tests/pix_util.py, pinned to the reference by
tests/test_oracle_pix_formats.py).  Also the misuse rules, the pipelined stitcher's input and output formats and
the C++ drop-in's file boundary next to the reference's codecs."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from openpano_b200.capi import LIB, PIX_GREY, PIX_RGB, PIX_RGB_PLANAR, PIX_RGBA, SRC_RGB8_DEV, Engine, PanoError
from tests import golden_util as gu
from tests import pix_util as xu

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "pix_formats_test"
CODE = {"grey": PIX_GREY, "rgb": PIX_RGB, "rgba": PIX_RGBA, "planar": PIX_RGB_PLANAR}
LAYOUTS = ["rgba", "planar"]


def _rgb(w, h, seed):
    return (synth.make_canvas(h, w, seed) * 255.0 + 0.5).astype(np.uint8)


def _lay(rgb, fmt, seed=0):
    """rgb (H×W×3) in layout fmt; RGBA gets a random fourth byte, grey takes the green channel."""
    if fmt == "rgba":
        return xu.to_rgba(rgb, alpha_seed=seed + 1)
    if fmt == "planar":
        return xu.to_planar(rgb)
    if fmt == "grey":
        return np.ascontiguousarray(rgb[..., 1])
    return rgb


def _hw(buf, fmt):
    return buf.shape[1:3] if fmt == "planar" else buf.shape[:2]


def _f32(orc, buf, fmt):
    """read_img's f32 image of a buffer, by the restatement."""
    if fmt == "rgba":
        return xu.orc_read_png_rgba(buf)
    if fmt == "planar":
        return xu.orc_read_img_planar(buf)
    return orc.read_img_rgb8(buf)


class _Dev:
    """Device buffers freed together."""

    def __init__(self, engine):
        self.eng, self.ptrs = engine, []

    def alloc(self, nbytes):
        p = self.eng.dev_alloc(max(nbytes, 256))
        self.ptrs.append(p)
        return p

    def upload(self, arr):
        p = self.alloc(arr.nbytes)
        self.eng.dev_upload(p, np.ascontiguousarray(arr))
        return p

    def free(self):
        for p in self.ptrs:
            self.eng.dev_free(p)
        self.ptrs = []


def _features(fs):
    out = []
    for i in range(fs.n_images):
        coor, desc = fs.download(i)
        real = np.zeros_like(coor)
        if len(coor):
            fs.eng._check(LIB.pano_featureset_download_real(fs._h, i, real.ctypes.data_as(C.POINTER(C.c_double))))
        out.append((coor, real, desc))
    fs.free()
    return out


def _same_features(a, b):
    return len(a) == len(b) and all(gu.same_bits(x, y) for fa, fb in zip(a, b) for x, y in zip(fa, fb))


def _sift_entries(engine, bufs, fmts, kinds=("pageable", "pinned", "device")):
    """The features of every 8-bit SIFT entry on buffers in formats fmts: host pageable (numpy, fmt=), host pinned
    and device pointers."""
    hw = [_hw(b, f) for b, f in zip(bufs, fmts)]
    ws, hs, codes = [s[1] for s in hw], [s[0] for s in hw], [CODE[f] for f in fmts]
    got = {}
    if "pageable" in kinds:
        got["pageable"] = _features(engine.sift_detect_batch_rgb8(bufs, fmt=list(fmts)))
    h_pix = [Engine.host_alloc(b.nbytes) for b in bufs]
    dev = _Dev(engine)
    try:
        for h, b in zip(h_pix, bufs):
            C.memmove(h, np.ascontiguousarray(b).ctypes.data, b.nbytes)
        d_pix = [dev.upload(b) for b in bufs]
        if "pinned" in kinds:
            got["pinned"] = _features(engine.sift_detect_batch_rgb8_ptr(h_pix, ws, hs, codes))
        if "device" in kinds:
            got["device"] = _features(engine.sift_detect_batch_rgb8_ptr(d_pix, ws, hs, codes, device=True))
    finally:
        for h in h_pix:
            Engine.host_free(h)
        dev.free()
    return got


# ----------------------------------------------------------------------------- SIFT
@pytest.mark.parametrize("fmt", LAYOUTS)
@pytest.mark.parametrize("w,h", [(1300, 867), (333, 517), (600, 400)])
def test_sift_layout_equals_interleaved(engine, fmt, w, h):
    rgb = _rgb(w, h, w + h)
    want = _features(engine.sift_detect_batch_rgb8([rgb]))
    assert len(want[0][0]) > 100
    for kind, got in _sift_entries(engine, [_lay(rgb, fmt, w)], [fmt]).items():
        assert _same_features(got, want), kind


def test_sift_alpha_bytes_change_nothing(engine):
    rgb = _rgb(640, 480, 3)
    a = _features(engine.sift_detect_batch_rgb8([xu.to_rgba(rgb)], fmt="rgba"))
    b = _features(engine.sift_detect_batch_rgb8([xu.to_rgba(rgb, alpha_seed=77)], fmt="rgba"))
    assert _same_features(a, b) and _same_features(a, _features(engine.sift_detect_batch_rgb8([rgb])))


def test_sift_mixed_batch_all_formats(engine, orc):
    """One batch of the four formats and different shapes, against sift_detect_batch on the restatement's f32
    images; a grey-valued RGBA image (a grey PNG) is divided by 255, unlike the same values as PANO_PIX_GREY."""
    fmts = ["grey", "rgba", "rgb", "planar", "rgba", "grey"]
    shapes = [(600, 400), (1300, 867), (333, 517), (1500, 1112), (517, 333), (640, 480)]
    bufs = [_lay(_rgb(w, h, 11 * k + 3), f, k) for k, ((w, h), f) in enumerate(zip(shapes, fmts))]
    grey = bufs[5]
    bufs[4] = np.ascontiguousarray(np.repeat(_lay(_rgb(517, 333, 9), "grey")[..., None], 4, axis=2))   # r = g = b
    bufs[4][..., 3] = 0
    f32 = [_f32(orc, b, f) for b, f in zip(bufs, fmts)]
    want = _features(engine.sift_detect_batch(f32))
    for kind, got in _sift_entries(engine, bufs, fmts).items():
        assert _same_features(got, want), kind
    g = bufs[4][..., 0]
    assert gu.same_bits(f32[4], (g.astype(np.float64) / 255.0).astype(np.float32)[..., None].repeat(3, 2))
    as_grey = _features(engine.sift_detect_batch_rgb8([np.ascontiguousarray(g)]))
    assert not _same_features(as_grey, [want[4]])
    assert _same_features(_features(engine.sift_detect_batch_rgb8([grey])), [want[5]])


def test_sift_capacity_growth_rereads_layouts(monkeypatch, orc):
    """Lists that start at 256 entries grow at the first count query: the batch (host and device) and a stream
    window read their RGBA and planar sources again."""
    rgb = [_rgb(1300, 867, 5), _rgb(1500, 1112, 6)]
    bufs, fmts = [_lay(rgb[0], "rgba", 1), _lay(rgb[1], "planar")], ["rgba", "planar"]
    monkeypatch.delenv("PANO_SIFT_CAP", raising=False)
    eng = Engine(0)
    try:
        want = _features(eng.sift_detect_batch_rgb8(rgb))
    finally:
        eng.close()
    assert max(len(f[0]) for f in want) > 256
    monkeypatch.setenv("PANO_SIFT_CAP", "256")
    for kind in ("pageable", "device", "stream"):
        eng = Engine(0)
        try:
            if kind == "stream":
                got = _features(eng.sift_lazy(bufs, window=[1, 1], fmt=fmts))
            else:
                got = _sift_entries(eng, bufs, fmts, (kind,))[kind]
        finally:
            eng.close()
        assert _same_features(got, want), kind


def _dev_stream_add(s, dev, bufs, fmt):
    s.add([dev.upload(b) for b in bufs], kind=SRC_RGB8_DEV, channels=CODE[fmt])


@pytest.mark.parametrize("windows", [[1, 1, 1, 1, 1], [2, 3], [5], [3, 1, 1]])
def test_sift_stream_layouts(engine, windows):
    """The stream over host and device windows, one format per window, windows differing in format."""
    rgb = [_rgb(w, h, 20 + k) for k, (w, h) in enumerate([(600, 400), (1300, 867), (333, 517), (640, 480), (517, 333)])]
    want = _features(engine.sift_detect_batch_rgb8(rgb))
    cycle = ["rgba", "planar", "rgb", "grey"]
    fmts = [cycle[q % 4] for q in range(len(windows))]
    if "grey" in fmts:
        want_grey = {k for q, f in enumerate(fmts) if f == "grey" for k in range(sum(windows[:q]), sum(windows[:q + 1]))}
        want = _features(engine.sift_detect_batch_rgb8([np.ascontiguousarray(x[..., 1]) if k in want_grey else x
                                                        for k, x in enumerate(rgb)]))
    bufs, k = [], 0
    for q, n in zip(fmts, windows):
        bufs.append([_lay(x, q, k + i) for i, x in enumerate(rgb[k:k + n])])
        k += n
    got_host = _features(engine.sift_lazy([b for win in bufs for b in win], window=windows, fmt=fmts))
    assert _same_features(got_host, want)
    s = engine.sift_stream([x.shape[:2] for x in rgb])
    dev = _Dev(engine)
    try:
        for win, q in zip(bufs, fmts):
            _dev_stream_add(s, dev, win, q)
        got_dev = _features(s.finish())
    finally:
        s.close()
        dev.free()
    assert _same_features(got_dev, want)


# ----------------------------------------------------------------------------- blend
def _stack(n, fmts):
    imgs, org = synth.make_stack(n, 240, 180, 70, 29, rows=2, step_y=60)
    rgb = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    items, geom = synth.translation_blend_setup(org, 240, 180)
    return rgb, [_lay(x, f, k) for k, (x, f) in enumerate(zip(rgb, fmts))], items, geom


def _blend_pair(engine, rgb, bufs, fmts, items, geom, bands, p, cuts=None):
    """(pano_blend_rgb8_dev of the interleaved pixels, of the buffers, the buffers' row strips concatenated)."""
    shapes = [x.shape[:2] for x in rgb]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    dev = _Dev(engine)
    try:
        d_rgb, d_buf = [dev.upload(x) for x in rgb], [dev.upload(b) for b in bufs]
        d_out = dev.alloc(tw * th * 12)
        want, got = np.empty((th, tw, 3), np.float32), np.empty((th, tw, 3), np.float32)
        engine.blend_rgb8_dev(d_rgb, [3] * len(rgb), shapes, items, geom, d_out, tw, th, bands, p)
        engine.dev_download(want, d_out)
        engine.blend_rgb8_dev(d_buf, [CODE[f] for f in fmts], shapes, items, geom, d_out, tw, th, bands, p)
        engine.dev_download(got, d_out)
        parts = []
        for r0, r1 in zip((cuts or [])[:-1], (cuts or [])[1:]):
            part = np.empty((r1 - r0, tw, 3), np.float32)
            engine.blend_rows_rgb8_dev(d_buf, [CODE[f] for f in fmts], shapes, items, geom, d_out, tw, th, r0, r1,
                                       bands, p)
            engine.dev_download(part, d_out)
            parts.append(part)
    finally:
        dev.free()
    return want, got, parts


@pytest.mark.parametrize("bands", [0, 5])
@pytest.mark.parametrize("fmts", [["rgba"] * 6, ["planar"] * 6, ["rgba", "planar", "rgb", "rgba", "planar", "rgb"]])
def test_blend_layouts_equal_interleaved(engine, orc, fmts, bands):
    p = default_params(multiband=max(bands, 1))
    rgb, bufs, items, geom = _stack(6, fmts)
    th = max(it[3] for it in items)
    want, got, parts = _blend_pair(engine, rgb, bufs, fmts, items, geom, bands, p, cuts=[0, 50, 51, 130, th])
    assert (want[..., 0] == -1).any() and (want[..., 0] >= 0).mean() > 0.5
    if bands == 0:
        assert gu.same_bits(want, orc.blend([orc.read_img_rgb8(x) for x in rgb], items, geom, 0, p))
    assert gu.same_bits(got, want)
    assert gu.same_bits(np.concatenate(parts), want)


@pytest.mark.parametrize("bands,lazy", [(0, 1), (0, 0), (3, 1)])
def test_blend_stream_layouts(engine, bands, lazy):
    """The blend stream from host and device windows whose formats differ."""
    p = default_params(multiband=max(bands, 1), lazy_read=lazy)
    windows, wfmts = [2, 1, 3], ["rgba", "planar", "rgba"]
    fmts = [f for n, f in zip(windows, wfmts) for _ in range(n)]
    rgb, bufs, items, geom = _stack(6, fmts)
    want, _, _ = _blend_pair(engine, rgb, rgb, ["rgb"] * 6, items, geom, bands, p)
    got = engine.blend_lazy(bufs, items, geom, bands, p, window=windows, fmt=wfmts)
    assert gu.same_bits(got, want)
    s = engine.blend_stream([x.shape[:2] for x in rgb], items, geom, bands, p)
    dev = _Dev(engine)
    try:
        k = 0
        for n, f in zip(windows, wfmts):
            _dev_stream_add(s, dev, bufs[k:k + n], f)
            k += n
        got_dev = s.finish()
    finally:
        s.close()
        dev.free()
    assert gu.same_bits(got_dev, want)


@pytest.mark.parametrize("bands", [0, 3])
def test_blend_stream_profile_names(engine, bands):
    """Each instantiation of the stream's source-reading kernel (k_linear_accumulate, k_mb_first_level) is profiled
    under its own name: f32 sources under the kernel's, grey and interleaved RGB under _rgb8, RGBA and planar under
    _pix8; one launch for a window of two images."""
    p = default_params(multiband=max(bands, 1))
    kernel = "k_mb_first_level" if bands else "k_linear_accumulate"
    rgb, _, items, geom = _stack(2, ["rgb"] * 2)
    dev = _Dev(engine)
    try:
        for fmt, name in (("f32", kernel), ("grey", kernel + "_rgb8"), ("rgb", kernel + "_rgb8"),
                          ("rgba", kernel + "_pix8"), ("planar", kernel + "_pix8")):
            s = engine.blend_stream([x.shape[:2] for x in rgb], items, geom, bands, p)
            try:
                engine.profile(True)
                engine.profile_reset()
                if fmt == "f32":
                    s.add([engine.read_img_rgb8(x) for x in rgb])
                else:
                    _dev_stream_add(s, dev, [_lay(x, fmt) for x in rgb], fmt)
                engine.sync()
                prof = engine.profile_read()
            finally:
                engine.profile(False)
                s.close()
            assert {k: v[0] for k, v in prof.items() if k.startswith(kernel)} == {name: 1}, (fmt, prof)
    finally:
        dev.free()


@pytest.mark.parametrize("kernel", ["k_linear_blend", "k_mb_first_level", "k_cyl_warp", "k_pyramid_grey"])
def test_batch_profile_names(engine, kernel):
    """The same for the batch entries' source-reading kernels (pano_blend_dev / pano_blend_rgb8_dev with 0 and 3
    bands, the batched cylinder warp, SIFT): one launch per batch, under _pix8 as soon as one image of the batch is
    RGBA or planar."""
    bands = 3 if kernel == "k_mb_first_level" else 0
    p = default_params(multiband=max(bands, 1))
    rgb, _, items, geom = _stack(2, ["rgb"] * 2)
    shapes = [x.shape[:2] for x in rgb]
    ws, hs = [w for _, w in shapes], [h for h, _ in shapes]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    outs = [engine.cyl_warp_shape(w, h, 1.0, p)[:2] for w, h in zip(ws, hs)]
    dev = _Dev(engine)
    try:
        d_out = dev.alloc(tw * th * 12)
        d_warp = [dev.alloc(ow * oh * 12) for ow, oh in outs]
        for fmts, name in ((None, kernel), (["grey"] * 2, kernel + "_rgb8"), (["rgb"] * 2, kernel + "_rgb8"),
                           (["rgba"] * 2, kernel + "_pix8"), (["planar"] * 2, kernel + "_pix8"),
                           (["rgb", "rgba"], kernel + "_pix8")):
            if fmts is None:
                d_src, codes = [dev.upload(engine.read_img_rgb8(x)) for x in rgb], None
            else:
                d_src, codes = [dev.upload(_lay(x, f)) for x, f in zip(rgb, fmts)], [CODE[f] for f in fmts]
            engine.profile(True)
            engine.profile_reset()
            try:
                fs = None
                if kernel == "k_cyl_warp":
                    if codes is None:
                        engine.cyl_warp_batch_dev(d_src, shapes, d_warp, None, 1.0, p)
                    else:
                        engine.cyl_warp_batch_rgb8_dev(d_src, codes, shapes, d_warp, None, 1.0, p)
                elif kernel == "k_pyramid_grey":
                    fs = (engine.sift_detect_batch_ptr(d_src, ws, hs, p, device=True) if codes is None
                          else engine.sift_detect_batch_rgb8_ptr(d_src, ws, hs, codes, p, device=True))
                elif codes is None:
                    engine.blend_dev(d_src, shapes, items, geom, d_out, tw, th, bands, p)
                else:
                    engine.blend_rgb8_dev(d_src, codes, shapes, items, geom, d_out, tw, th, bands, p)
                engine.sync()
                prof = engine.profile_read()
            finally:
                engine.profile(False)
            if fs is not None:
                fs.free()
            assert {k: v[0] for k, v in prof.items() if k.startswith(kernel)} == {name: 1}, (fmts, prof)
    finally:
        dev.free()


# ----------------------------------------------------------------------------- cylinder warp, conversion
@pytest.mark.parametrize("hf", [1.0, 1.2])
def test_cyl_warp_layouts_equal_interleaved(engine, hf):
    shapes = [(333, 217), (240, 180), (50, 3), (3, 50), (600, 400)]
    fmts = ["rgba", "planar", "rgba", "planar", "rgb"]
    rgb = [_rgb(w, h, 30 + k) for k, (w, h) in enumerate(shapes)]
    bufs = [_lay(x, f, k) for k, (x, f) in enumerate(zip(rgb, fmts))]
    rng = np.random.RandomState(4)
    kpts = [np.ascontiguousarray((rng.rand(20, 2) - 0.5) * np.array([w * 1.1, h * 1.1]), np.float64) for w, h in shapes]
    p = default_params()
    outs = [engine.cyl_warp_shape(w, h, hf, p)[:2] for w, h in shapes]
    hw = [x.shape[:2] for x in rgb]
    dev = _Dev(engine)
    try:
        d_rgb, d_buf = [dev.upload(x) for x in rgb], [dev.upload(b) for b in bufs]
        d_a, d_b = [dev.alloc(ow * oh * 12) for ow, oh in outs], [dev.alloc(ow * oh * 12) for ow, oh in outs]
        ka, kb = [k.copy() for k in kpts], [k.copy() for k in kpts]
        engine.cyl_warp_batch_rgb8_dev(d_rgb, [3] * len(rgb), hw, d_a, ka, hf, p)
        engine.cyl_warp_batch_rgb8_dev(d_buf, [CODE[f] for f in fmts], hw, d_b, kb, hf, p)
        for (ow, oh), a, b, k in zip(outs, d_a, d_b, range(len(outs))):
            wa, gb = np.empty((oh, ow, 3), np.float32), np.empty((oh, ow, 3), np.float32)
            engine.dev_download(wa, a)
            engine.dev_download(gb, b)
            assert gu.same_bits(gb, wa), f"warp of image {k}"
            assert (wa >= 0).any()
    finally:
        dev.free()
    assert all(gu.same_bits(a, b) for a, b in zip(ka, kb))


@pytest.mark.parametrize("w,h", [(2, 2), (3, 50), (50, 3), (333, 217), (7, 5)])
def test_rgb8_to_mat32f_layouts(engine, orc, w, h):
    """Every format in one batch and on its own, against the restatement; RGBA rows of 4w bytes are not multiples
    of 16 for these widths."""
    rgb = _rgb(w, h, w * 3 + h)
    fmts = ["rgba", "planar", "rgb", "grey"]
    bufs = [_lay(rgb, f, 5) for f in fmts]
    want = [_f32(orc, b, f) for b, f in zip(bufs, fmts)]
    assert gu.same_bits(want[0], want[2]) and gu.same_bits(want[1], want[2])
    dev = _Dev(engine)
    try:
        d_in = [dev.upload(b) for b in bufs]
        d_out = [dev.alloc(w * h * 12) for _ in bufs]
        for single in (False, True):
            if single:
                for d, f, o in zip(d_in, fmts, d_out):
                    engine.rgb8_to_mat32f_dev(d, w, h, CODE[f], o)
            else:
                engine.rgb8_to_mat32f_batch_dev(d_in, [w] * 4, [h] * 4, [CODE[f] for f in fmts], d_out)
            for o, x in zip(d_out, want):
                got = np.empty((h, w, 3), np.float32)
                engine.dev_download(got, o)
                assert gu.same_bits(got, x)
    finally:
        dev.free()
    for f, b, x in zip(fmts, bufs, want):
        assert gu.same_bits(engine.read_img_rgb8(b, fmt=None if f in ("rgb", "grey") else f), x)


@pytest.mark.parametrize("shape", [(2, 2), (3, 50), (50, 3)])
def test_small_shape_blends_of_layouts(engine, shape):
    """The smallest and thinnest sources the blend takes, one image per blend, in both layouts."""
    w, h = shape
    rgb = [_rgb(w, h, 61)]
    items, geom = synth.translation_blend_setup([(0, 0)], w, h)
    for f in LAYOUTS:
        for bands in (0, 2):
            p = default_params(multiband=max(bands, 1))
            want, got, _ = _blend_pair(engine, rgb, [_lay(rgb[0], f, 2)], [f], items, geom, bands, p)
            assert gu.same_bits(got, want), (f, bands)
            if min(w, h) > 2:
                assert (want >= 0).any(), (f, bands)


# ----------------------------------------------------------------------------- output conversion
def _mosaic(engine):
    rgb, _, items, geom = _stack(5, ["rgb"] * 5)
    return engine.blend_lazy(rgb, items, geom, 0)


@pytest.mark.parametrize("crop", [True, False])
def test_mat32f_to_pix8_formats(engine, orc, crop):
    """write_rgb's conversion into each layout, with and without crop's rectangle, on a blend output with
    Color::NO pixels and on a small odd-sized mosaic."""
    for mat in (_mosaic(engine), xu.mosaic_with_holes(37, 29, seed=3)):
        assert (mat < 0).any()
        if crop:
            want_rect, sub = orc.crop(mat)
        else:
            want_rect, sub = None, mat
        rgb = orc.write_rgb8(sub)
        want = {"rgb": rgb, "rgba": xu.orc_write_png_rgba(sub), "planar": xu.orc_write_rgb_planar(sub)}
        assert np.array_equal(want["rgba"], xu.to_rgba(rgb)) and np.array_equal(want["planar"], xu.to_planar(rgb))
        for fmt in ("rgb", "rgba", "planar"):
            rect, px = engine.crop_write_pix8(mat, crop=crop, fmt=fmt)
            if crop:
                assert np.array_equal(rect, want_rect)
            assert np.array_equal(px, want[fmt]), fmt


# ----------------------------------------------------------------------------- misuse
BAD_FORMATS = [0, 2, 4, 5, 0x103, 0x204]


def test_invalid_formats_and_alignment(engine, orc):
    """Unknown formats and a misaligned device RGBA pointer return PANO_ERR_INVALID with a message and launch
    nothing; the context gives correct results afterwards."""
    vp, ip = C.c_void_p, C.c_int
    p = default_params()
    rgb, bufs, items, geom = _stack(3, ["rgba"] * 3)
    n = len(rgb)
    ws, hs = [x.shape[1] for x in rgb], [x.shape[0] for x in rgb]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    ow, oh = engine.cyl_warp_shape(240, 180, 1.0, p)[:2]

    def arr(t, vals):
        return (t * max(len(vals), 1))(*vals)

    dev = _Dev(engine)
    try:
        d_buf = [dev.upload(b) for b in bufs]
        d_mis = [d_buf[0], d_buf[1] + 1, d_buf[2]]                    # a 1-byte offset: not 4-byte aligned
        d_out = dev.alloc(tw * th * 12)
        d_warp = [dev.alloc(ow * oh * 12) for _ in range(n)]
        blend_args, g = engine._blend_args([None] * n, [x.shape[:2] for x in rgb], items, geom)
        fs = C.c_void_p()
        host = [b.ctypes.data for b in bufs]

        jobs = engine._cyl_jobs([None] * n, [x.shape[:2] for x in rgb], d_warp, None, 1.0, p)

        def calls(ptrs, ch):
            """(name, call) of every 8-bit device entry on sources ptrs in formats ch; a stream is created before
            its call, so that its own launches are not counted."""
            yield "sift dev", lambda: LIB.pano_sift_detect_batch_rgb8_dev(
                engine._h, n, arr(vp, ptrs), arr(ip, ws), arr(ip, hs), arr(ip, ch), C.byref(p), C.byref(fs))
            yield "blend", lambda: LIB.pano_blend_rgb8_dev(engine._h, n, blend_args, arr(vp, ptrs), arr(ip, ch),
                                                           C.byref(g), 0, C.byref(p), vp(d_out), tw, th)
            yield "rows", lambda: LIB.pano_blend_rows_rgb8_dev(engine._h, n, blend_args, arr(vp, ptrs), arr(ip, ch),
                                                               C.byref(g), 3, C.byref(p), vp(d_out), tw, th, 10, 40)
            yield "warp", lambda: LIB.pano_cyl_warp_batch_rgb8_dev(engine._h, n, jobs, arr(vp, ptrs), arr(ip, ch), 1.0,
                                                                   C.byref(p))
            yield "convert", lambda: LIB.pano_rgb8_to_mat32f_batch_dev(engine._h, n, arr(vp, ptrs), arr(ip, ws),
                                                                       arr(ip, hs), arr(ip, ch), arr(vp, [d_out] * n))
            for name in ("sift stream", "blend stream"):
                shapes = [x.shape[:2] for x in rgb]
                st = engine.sift_stream(shapes) if name == "sift stream" else engine.blend_stream(shapes, items, geom)
                try:
                    yield name, lambda: type(st)._ADD(st._h, 0, n, arr(vp, ptrs), SRC_RGB8_DEV, ch[1])
                finally:
                    st.close()

        def refused(call, word, what):
            before = engine.launch_count()
            assert call() == -2, what
            assert word in LIB.pano_last_error(engine._h).decode(), what
            assert engine.launch_count() == before, what

        for bad in BAD_FORMATS:
            for name, call in calls(d_buf, [PIX_RGBA, bad, PIX_RGBA]):
                refused(call, "format", (name, bad))
            refused(lambda: LIB.pano_sift_detect_batch_rgb8(engine._h, n, arr(vp, host), arr(ip, ws), arr(ip, hs),
                                                            arr(ip, [3, bad, 3]), C.byref(p), C.byref(fs)),
                    "format", ("sift host", bad))
        for name, call in calls(d_mis, [PIX_RGBA] * n):
            refused(call, "aligned", name)
        for bad in [0, 1, 4, 0x204]:
            refused(lambda: LIB.pano_mat32f_to_pix8_dev(engine._h, vp(d_out), tw, th, None, bad, vp(d_warp[0])),
                    "format", ("output", bad))
        with pytest.raises(PanoError):
            engine.sift_detect_batch_rgb8([bufs[0]])                  # H×W×4 without fmt="rgba"
        with pytest.raises(PanoError):
            engine.sift_detect_batch_rgb8([rgb[0]], fmt="planar")
    finally:
        dev.free()
    # the context is still usable and correct
    want = _features(engine.sift_detect_batch([orc.read_img_rgb8(x) for x in rgb]))
    assert _same_features(_features(engine.sift_detect_batch_rgb8(bufs, fmt="rgba")), want)
    w_blend, g_blend, _ = _blend_pair(engine, rgb, bufs, ["rgba"] * n, items, geom, 0, p)
    assert gu.same_bits(g_blend, w_blend)


# ----------------------------------------------------------------------------- stitcher, C++ drop-in
def _stitch(rgb, fmt_in, fmt_out, pairs, items, geom, p):
    from openpano_b200.stitcher import PipelinedStitcher, unpack_rgb8_mosaic
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    bufs = [_lay(x, fmt_in, k) for k, x in enumerate(rgb)]
    ps = PipelinedStitcher(0, p, depth=2, rgb8=True, crop=True, in_format=fmt_in, out_format=fmt_out)
    try:
        assert ps.in_bytes([x.shape[:2] for x in rgb]) == sum(b.nbytes for b in bufs)
        out = np.zeros(ps.out_bytes((ow, oh)), np.uint8)
        k = ps.stage([b.ctypes.data for b in bufs], [x.shape[:2] for x in rgb], (ow, oh))
        matches = ps.wait(ps.run(k, pairs, items, geom, out.ctypes.data))
    finally:
        ps.close()
    rect, px = unpack_rgb8_mosaic(out, (ow, oh), cropped=True, out_format=fmt_out)
    return rect, px.copy(), matches


def test_pipelined_stitcher_formats(orc):
    from openpano_b200.stitcher import ordered_pairs
    imgs, org = synth.make_stack(4, 900, 700, 300, 2)
    rgb = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    items, geom = synth.translation_blend_setup(org, 900, 700)
    p = default_params(ordered_input=1)
    pairs = ordered_pairs(len(rgb))
    rect, px, matches = _stitch(rgb, "rgb", "rgb", pairs, items, geom, p)
    want_rect, want = orc.crop(orc.blend([orc.read_img_rgb8(x) for x in rgb], items, geom, 0, p))
    assert np.array_equal(rect, want_rect) and np.array_equal(px, orc.write_rgb8(want))
    relaid = {"rgb": px, "rgba": xu.to_rgba(px), "planar": xu.to_planar(px)}
    for fin, fout in [("rgba", "rgb"), ("planar", "rgb"), ("rgb", "rgba"), ("rgb", "planar"), ("rgba", "planar"),
                      ("planar", "rgba")]:
        r, got, m = _stitch(rgb, fin, fout, pairs, items, geom, p)
        assert np.array_equal(r, rect), (fin, fout)
        assert np.array_equal(got, relaid[fout]), (fin, fout)
        assert len(m) == len(matches) and all(np.array_equal(a, b) for a, b in zip(m, matches)), (fin, fout)


def test_cpp_file_boundary_equals_reference_codecs(tmp_path):
    """load_pixels / B200PixelBlender / write_mosaic (openpano_b200/host/pano_host_io.hh) next to read_img, the
    reference's detector and blenders and write_rgb on PNG files of every colour type, a PPM and a PGM
    (oracle/_ref/pix_formats_test)."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/pix_formats_test not built (needs the reference sources at build time)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(tmp_path)], capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "PIX FORMATS TEST OK" in out.stdout
    assert out.stdout.count("identical") == 9 + 8 + 2
