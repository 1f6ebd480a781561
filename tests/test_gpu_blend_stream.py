"""GPU: the blend stream (pano_blend_stream_*, LAZY_READ's memory contract).  The mosaic must have the raw
bits of pano_blend on the f32 images for every window partition and source kind, 8-bit sources included
(read_img's conversion of each tap), and a stream must never hold more than the canvas state plus two
windows of sources.  Also the misuse rules and the C++ adaptor (B200LazyBlender) next to the reference's
own LinearBlender / MultiBandBlender."""
import ctypes as C
import os
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests import golden_util as gu
from tests.test_gpu_match_warp_blend import _perspective_items

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "lazy_blend_test"
MB = 1 << 20


def _pix(imgs):
    return [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]


def _partition(name, n):
    return {"ones": [1] * n, "threes": [3] * (n // 3) + ([n % 3] if n % 3 else []), "all": [n],
            "irregular": [2, n - 3, 1]}[name]


def _stack(n=7):
    imgs, org = synth.make_stack(n, 240, 180, 70, 23, rows=2, step_y=60)
    items, geom = synth.translation_blend_setup(org, 240, 180)
    return imgs, items, geom


@pytest.mark.parametrize("lazy,ordered", [(1, 0), (1, 1), (0, 0), (0, 1)])
def test_linear_stream_equals_blend_and_reference(engine, orc, lazy, ordered):
    imgs, items, geom = _stack(5)
    pix = _pix(imgs)
    p = default_params(lazy_read=lazy, ordered_input=ordered)
    f32 = [orc.read_img_rgb8(x) for x in pix]
    want = engine.blend(f32, items, geom, 0, p)
    assert gu.same_bits(want, orc.blend(f32, items, geom, 0, p))
    for window in ([2, 3], 1, [5]):
        assert gu.same_bits(engine.blend_lazy(pix, items, geom, 0, p, window), want), window
        assert gu.same_bits(engine.blend_lazy(f32, items, geom, 0, p, window), want), window


@pytest.mark.parametrize("bands", [0, 1, 2, 3, 5])
@pytest.mark.parametrize("part", ["ones", "threes", "all", "irregular"])
def test_stream_partitions_bit_exact(engine, bands, part):
    imgs, items, geom = _stack(7)
    pix = _pix(imgs)
    f32 = [engine.read_img_rgb8(x) for x in pix]
    window = _partition(part, len(imgs))
    assert sum(window) == len(imgs)
    want = engine.blend(f32, items, geom, bands)
    assert (want[..., 0] == -1).any() and (want[..., 0] >= 0).mean() > 0.5
    assert gu.same_bits(engine.blend_lazy(pix, items, geom, bands, None, window), want)


@pytest.mark.parametrize("projection", [0, 1, 2])
@pytest.mark.parametrize("bands", [0, 3])
def test_stream_projections_bit_exact(engine, orc, projection, bands):
    imgs, org = synth.make_stack(4, 300, 200, 100, 7)
    items, geom = _perspective_items(org, 4, projection)
    pix = _pix(imgs)
    f32 = [orc.read_img_rgb8(x) for x in pix]
    want = engine.blend(f32, items, geom, bands)
    assert (want < 0).mean() < 0.9
    assert gu.same_bits(want, orc.blend(f32, items, geom, bands))
    for window in (1, [3, 1]):
        assert gu.same_bits(engine.blend_lazy(pix, items, geom, bands, None, window), want)


@pytest.mark.parametrize("bands", [0, 3])
def test_all_source_kinds(engine, bands):
    """Device and host sources, f32 and 8-bit, pageable and pinned host buffers, mixed across windows."""
    from openpano_b200.capi import SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_DEV, SRC_RGB8_HOST, Engine
    imgs, items, geom = _stack(8)
    pix = _pix(imgs)
    f32 = [engine.read_img_rgb8(x) for x in pix]
    want = engine.blend(f32, items, geom, bands)
    shapes = [im.shape[:2] for im in imgs]
    d_f32 = [engine.dev_alloc(x.nbytes) for x in f32]
    d_pix = [engine.dev_alloc(x.nbytes) for x in pix]
    h_f32 = [Engine.host_alloc(x.nbytes) for x in f32]
    h_pix = [Engine.host_alloc(x.nbytes) for x in pix]
    try:
        for d, h, x in zip(d_f32 + d_pix, h_f32 + h_pix, f32 + pix):
            engine.dev_upload(d, x)
            C.memmove(h, x.ctypes.data, x.nbytes)
        s = engine.blend_stream(shapes, items, geom, bands)
        try:
            s.add(d_f32[0:2], SRC_F32_DEV)
            s.add(h_pix[2:3], SRC_RGB8_HOST)             # pinned
            s.add(f32[3:4])                               # pageable f32
            s.add(d_pix[4:6], SRC_RGB8_DEV)
            s.add(h_f32[6:7], SRC_F32_HOST)              # pinned
            s.add(pix[7:8])                               # pageable u8
            got = s.finish()
        finally:
            s.close()
        assert gu.same_bits(got, want)
        for kind, ptrs in ((SRC_F32_DEV, d_f32), (SRC_F32_HOST, h_f32), (SRC_RGB8_DEV, d_pix), (SRC_RGB8_HOST, h_pix)):
            s = engine.blend_stream(shapes, items, geom, bands)
            d_out = engine.dev_alloc(want.nbytes)
            try:
                for k in range(0, 8, 3):
                    s.add(ptrs[k:k + 3], kind)
                s.finish_dev(d_out)
                got = np.empty_like(want)
                engine.dev_download(got, d_out)
            finally:
                s.close()
                engine.dev_free(d_out)
            assert gu.same_bits(got, want), kind
    finally:
        for d in d_f32 + d_pix:
            engine.dev_free(d)
        for h in h_f32 + h_pix:
            Engine.host_free(h)


@pytest.mark.parametrize("bands", [0, 2])
def test_grey_sources(engine, orc, bands):
    """channels == 1: read_img replicates the grey value without dividing it (imgio.cc:84-87)."""
    imgs, items, geom = _stack(5)
    grey = [x[..., 1].copy() for x in _pix(imgs)]
    f32 = [orc.read_img_rgb8(x) for x in grey]
    assert f32[0].max() > 1.0
    want = engine.blend(f32, items, geom, bands)
    assert gu.same_bits(want, orc.blend(f32, items, geom, bands))
    assert gu.same_bits(engine.blend_lazy(grey, items, geom, bands, None, [2, 3]), want)
    assert gu.same_bits(engine.blend_lazy([g[..., None] for g in grey], items, geom, bands, None, 5), want)


@pytest.mark.parametrize("bands", [0, 3])
def test_window_over_64_images_on_one_tile(engine, bands):
    """70 images cover the same tiles: the per-tile list overflows and the pixel loop walks the whole window."""
    imgs, org = synth.make_stack(70, 64, 48, 1, 31)
    items, geom = synth.translation_blend_setup(org, 64, 48)
    pix = _pix(imgs)
    f32 = [engine.read_img_rgb8(x) for x in pix]
    for lazy in (1, 0):
        p = default_params(lazy_read=lazy)
        want = engine.blend(f32, items, geom, bands, p)
        assert gu.same_bits(engine.blend_lazy(pix, items, geom, bands, p, [70]), want)
        assert gu.same_bits(engine.blend_lazy(pix, items, geom, bands, p, [66, 4]), want)


def _canvas_state(items, tw, th, bands):
    """The stream's canvas state as include/pano_b200.h states it (finish()'s output included)."""
    if bands == 0:
        return 16 * tw * th
    roi = sum(-(-(x1 - x0 + 1) // 32) * 32 * (y1 - y0 + 1) for x0, y0, x1, y1, _ in items)
    return 33 * roi + tw * th + 12 * tw * th


@pytest.mark.parametrize("bands", [0, 5])
def test_memory_bound(monkeypatch, bands):
    """1 GB of 8-bit sources streamed two at a time: the pool's high-water mark stays within the canvas state plus
    two windows plus 64 MB, and below the resident path's (8-bit and f32 copies of every image on the device, then
    pano_blend_dev) by at least the f32 source bytes.  Both give the same bits."""
    from openpano_b200.capi import Engine
    monkeypatch.setenv("PANO_CACHE_MB", "0")
    w, h, n = 2000, 1500, 120
    base = np.random.RandomState(3).randint(0, 256, (h + 7 * 750, w + 14 * 1000, 3)).astype(np.uint8)
    org = [(c * 1000, r * 750) for r in range(8) for c in range(15)]
    pix = [np.ascontiguousarray(base[y:y + h, x:x + w]) for x, y in org]
    items, geom = synth.translation_blend_setup(org, w, h)
    src_u8 = sum(x.nbytes for x in pix)
    assert src_u8 >= 1 << 30
    eng = Engine(0)
    try:
        eng.trim()
        eng.sync()
        eng.mem_high_water(reset=True)
        s = eng.blend_stream([x.shape[:2] for x in pix], items, geom, bands)
        try:
            for k in range(0, n, 2):
                s.add(pix[k:k + 2])
            got = s.finish()
        finally:
            s.close()
        eng.sync()
        stream_mark = eng.mem_high_water(reset=True)
        th, tw = got.shape[:2]
        bound = _canvas_state(items, tw, th, bands) + 2 * 2 * pix[0].nbytes + 64 * MB
        assert stream_mark <= bound, (stream_mark / MB, bound / MB)

        d_pix = [eng.dev_alloc(x.nbytes) for x in pix]
        d_f32 = [eng.dev_alloc(x.nbytes * 4) for x in pix]
        d_out = eng.dev_alloc(got.nbytes)
        want = np.empty_like(got)
        try:
            for d, x in zip(d_pix, pix):
                eng.dev_upload(d, x)
            eng.rgb8_to_mat32f_batch_dev(d_pix, [w] * n, [h] * n, [3] * n, d_f32)
            eng.blend_dev(d_f32, [x.shape[:2] for x in pix], items, geom, d_out, tw, th, bands)
            eng.dev_download(want, d_out)
        finally:
            for d in d_pix + d_f32 + [d_out]:
                eng.dev_free(d)
        eng.sync()
        resident_mark = eng.mem_high_water()
        assert gu.same_bits(got, want)
        assert resident_mark - stream_mark >= 4 * src_u8, (resident_mark / MB, stream_mark / MB, 4 * src_u8 / MB)
        print(f"bands={bands}: stream {stream_mark / MB:.0f} MB (bound {bound / MB:.0f} MB), "
              f"resident {resident_mark / MB:.0f} MB, 8-bit sources {src_u8 / MB:.0f} MB")
    finally:
        eng.close()


def test_misuse_is_invalid_and_sticky(engine, orc):
    from openpano_b200.capi import LIB, PanoError, SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_HOST
    imgs, items, geom = _stack(4)
    pix = _pix(imgs)
    shapes = [x.shape[:2] for x in pix]
    arr, g = engine._blend_args([None] * 4, shapes, items, geom)
    p = default_params()
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    out = np.empty((th, tw, 3), np.float32)
    fp = C.POINTER(C.c_float)

    def srcs(k0, k1):
        return (C.c_void_p * max(k1 - k0, 1))(*[x.ctypes.data for x in pix[k0:k1]])

    def fresh():
        h = C.c_void_p()
        assert LIB.pano_blend_stream_create(engine._h, 4, arr, C.byref(g), 0, C.byref(p), tw, th, C.byref(h)) == 0
        return h

    add = LIB.pano_blend_stream_add
    cases = {
        "out of order": lambda h: add(h, 1, 1, srcs(1, 2), SRC_RGB8_HOST, 3),
        "overlapping": lambda h: (add(h, 0, 2, srcs(0, 2), SRC_RGB8_HOST, 3), add(h, 1, 1, srcs(1, 2), SRC_RGB8_HOST, 3))[1],
        "excess": lambda h: add(h, 0, 5, srcs(0, 4), SRC_RGB8_HOST, 3),
        "empty": lambda h: add(h, 0, 0, srcs(0, 1), SRC_RGB8_HOST, 3),
        "finish early": lambda h: (add(h, 0, 3, srcs(0, 3), SRC_RGB8_HOST, 3), LIB.pano_blend_stream_finish(h, out.ctypes.data_as(fp)))[1],
        "u8 channels": lambda h: add(h, 0, 1, srcs(0, 1), SRC_RGB8_HOST, 2),
        "f32 channels": lambda h: add(h, 0, 1, srcs(0, 1), SRC_F32_HOST, 1),
        "unknown kind": lambda h: add(h, 0, 1, srcs(0, 1), 7, 3),
        "null list": lambda h: add(h, 0, 1, None, SRC_RGB8_HOST, 3),
        "null source": lambda h: add(h, 0, 1, (C.c_void_p * 1)(None), SRC_F32_DEV, 3),
        "null output": lambda h: (add(h, 0, 4, srcs(0, 4), SRC_RGB8_HOST, 3), LIB.pano_blend_stream_finish_dev(h, None))[1],
        "finish twice": lambda h: (add(h, 0, 4, srcs(0, 4), SRC_RGB8_HOST, 3), LIB.pano_blend_stream_finish(h, out.ctypes.data_as(fp)),
                                   LIB.pano_blend_stream_finish(h, out.ctypes.data_as(fp)))[2],
        "add after finish": lambda h: (add(h, 0, 4, srcs(0, 4), SRC_RGB8_HOST, 3), LIB.pano_blend_stream_finish(h, out.ctypes.data_as(fp)),
                                       add(h, 4, 1, srcs(0, 1), SRC_RGB8_HOST, 3))[2],
    }
    for name, call in cases.items():
        h = fresh()
        try:
            assert call(h) == -2, name
            assert add(h, 0, 1, srcs(0, 1), SRC_RGB8_HOST, 3) == -2, f"{name}: not sticky"
            assert LIB.pano_blend_stream_finish(h, out.ctypes.data_as(fp)) == -2, f"{name}: not sticky"
        finally:
            LIB.pano_blend_stream_free(h)
    h = C.c_void_p()
    assert LIB.pano_blend_stream_create(None, 4, arr, C.byref(g), 0, C.byref(p), tw, th, C.byref(h)) == -2
    assert LIB.pano_blend_stream_create(engine._h, 4, arr, C.byref(g), 0, C.byref(p), tw, th, None) == -2
    assert LIB.pano_blend_stream_create(engine._h, 4, arr, C.byref(g), 0, C.byref(p), tw + 1, th, C.byref(h)) == -2
    assert LIB.pano_blend_stream_add(None, 0, 1, srcs(0, 1), SRC_RGB8_HOST, 3) == -2
    assert LIB.pano_blend_stream_finish(None, out.ctypes.data_as(fp)) == -2
    LIB.pano_blend_stream_free(None)
    # the binding checks numpy shapes against the stream's and is sticky as well
    s = engine.blend_stream(shapes, items, geom, 0)
    try:
        with pytest.raises(PanoError) as ei:
            s.add([pix[0][:-1]])
        assert ei.value.code == -2
        with pytest.raises(PanoError):
            s.add(pix[0:1])
    finally:
        s.close()
    # the context is still usable
    f32 = [orc.read_img_rgb8(x) for x in pix]
    assert gu.same_bits(engine.blend_lazy(pix, items, geom, 0, None, 2), orc.blend(f32, items, geom, 0))


def test_cpp_lazy_blender_equals_reference_blenders(tmp_path):
    """B200LazyBlender (openpano_b200/host/pano_host.hh) next to the reference's LinearBlender (LAZY_READ 1 and 0)
    and MultiBandBlender, compiled against the reference's headers (oracle/_ref/lazy_blend_test)."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/lazy_blend_test not built (needs the reference sources at build time)")
    imgs, org = synth.make_stack(6, 200, 150, 60, 53, rows=2, step_y=50)
    items, geom = synth.translation_blend_setup(org, 200, 150)
    path = tmp_path / "stack.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<3i", len(imgs), 200, 150))
        for im in imgs:
            f.write(np.ascontiguousarray(im, np.float32).tobytes())
        for it in items:
            f.write(struct.pack("<4i", *it[:4]))
            f.write(struct.pack("<9d", *it[4]))
        f.write(struct.pack("<3d", geom["res_x"], geom["proj_min_x"], geom["proj_min_y"]))
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(path)], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "LAZY BLEND TEST OK" in out.stdout
    assert out.stdout.count("identical") == 12
