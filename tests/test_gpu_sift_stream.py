"""GPU: the SIFT stream (pano_sift_stream_*, LAZY_READ's feature stage).  For every window partition and source
kind the featureset must have the raw bits of pano_sift_detect_batch[_rgb8]'s (counts, coordinates, real
coordinates, descriptors, and so the match lists), a list overflow inside a window must re-run that window alone,
one stream must take more images than one SIFT batch, and a stream must never hold more than one window's SIFT
buffers plus two windows of sources plus the packed rows.  Also the misuse rules and the C++ adaptor
(B200SIFTDetector::detect_lazy) next to the reference's calc_feature loop."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests import golden_util as gu

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "lazy_sift_test"
MB = 1 << 20


def _pix(imgs):
    return [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]


def _real(fs, i):
    from openpano_b200.capi import LIB
    out = np.zeros((fs.count(i), 2), np.float64)
    fs.eng._check(LIB.pano_featureset_download_real(fs._h, i, out.ctypes.data_as(C.POINTER(C.c_double))))
    return out


def _assert_same(got, want, n, got_at=0, want_at=0):
    """Images got_at.. of `got` against want_at.. of `want`, bit for bit."""
    for i in range(n):
        assert got.count(got_at + i) == want.count(want_at + i), i
        gc, gd = got.download(got_at + i)
        wc, wd = want.download(want_at + i)
        assert gu.same_bits(gc, wc) and gu.same_bits(gd, wd), i
        assert gu.same_bits(_real(got, got_at + i), _real(want, want_at + i)), i


def _all_pairs(n):
    return [(i, j) for i in range(n) for j in range(i + 1, n)]


def _same_matches(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.fixture(scope="module")
def stack14():
    """A 13-image stack plus one 1500×1112 image (config 2's shape)."""
    imgs, _ = synth.make_stack(13, 400, 300, 110, 11)
    return imgs + [synth.make_canvas(1112, 1500, 12)]


@pytest.mark.parametrize("window", [1, [1, 4, 2, 3, 1, 3], 14])
def test_partitions_equal_batch(engine, stack14, window):
    imgs = stack14
    want = engine.sift_detect_batch(imgs)
    got = engine.sift_lazy(imgs, window)
    try:
        assert min(want.count(i) for i in range(14)) > 20
        _assert_same(got, want, 14)
        pairs = _all_pairs(14)
        m = engine.match_pairs(want, pairs)
        assert sum(len(x) for x in m) > 0
        assert _same_matches(engine.match_pairs(got, pairs), m)
    finally:
        got.free()
        want.free()


def test_all_source_kinds(engine):
    """Device and host sources, f32 and 8-bit, pageable and pinned host buffers, grey and colour windows."""
    from openpano_b200.capi import SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_DEV, SRC_RGB8_HOST, Engine
    imgs, _ = synth.make_stack(8, 360, 270, 100, 21)
    pix = _pix(imgs)
    for k in (2, 7):
        pix[k] = pix[k][..., 1].copy()          # grey: read_img replicates the value without dividing it
    chans = [1 if x.ndim == 2 else 3 for x in pix]
    f32 = [engine.read_img_rgb8(x) for x in pix]
    want = engine.sift_detect_batch_rgb8(pix)
    shapes = [x.shape[:2] for x in pix]
    d_f32 = [engine.dev_alloc(x.nbytes) for x in f32]
    d_pix = [engine.dev_alloc(x.nbytes) for x in pix]
    h_f32 = [Engine.host_alloc(x.nbytes) for x in f32]
    h_pix = [Engine.host_alloc(x.nbytes) for x in pix]
    try:
        for d, h, x in zip(d_f32 + d_pix, h_f32 + h_pix, f32 + pix):
            engine.dev_upload(d, x)
            C.memmove(h, x.ctypes.data, x.nbytes)
        s = engine.sift_stream(shapes)
        try:
            s.add(d_f32[0:2], SRC_F32_DEV)
            s.add(h_pix[2:3], SRC_RGB8_HOST, 1)          # pinned, grey
            s.add(f32[3:4])                               # pageable f32
            s.add(d_pix[4:6], SRC_RGB8_DEV, 3)
            s.add(h_f32[6:7], SRC_F32_HOST)              # pinned
            s.add(pix[7:8])                               # pageable u8, grey
            got = s.finish()
        finally:
            s.close()
        _assert_same(got, want, 8)
        got.free()
        for kind, ptrs in ((SRC_F32_DEV, d_f32), (SRC_F32_HOST, h_f32), (SRC_RGB8_DEV, d_pix), (SRC_RGB8_HOST, h_pix)):
            s = engine.sift_stream(shapes)
            try:
                k = 0
                for q in (2, 1, 4, 1):                    # windows of one channel count
                    s.add(ptrs[k:k + q], kind, chans[k] if kind in (SRC_RGB8_DEV, SRC_RGB8_HOST) else 3)
                    k += q
                got = s.finish()
            finally:
                s.close()
            _assert_same(got, want, 8)
            got.free()
    finally:
        want.free()
        for d in d_f32 + d_pix:
            engine.dev_free(d)
        for h in h_f32 + h_pix:
            Engine.host_free(h)


def test_list_growth_inside_a_window(engine, monkeypatch):
    """PANO_SIFT_CAP=256: the middle window holds an image whose lists overflow.  That window is run again with
    doubled lists before its sources leave, and the windows after it start from the larger lists."""
    from openpano_b200.capi import Engine
    busy, _ = synth.make_stack(3, 480, 360, 160, 43)
    quiet = []
    for k in (1, 2, 3):                                  # a gradient and three discs: few keypoints
        im = np.empty((300, 400, 3), np.float32)
        im[...] = (np.linspace(0.2, 0.7, 400, dtype=np.float32)[None, :, None] + 0.1 * k) % 1.0
        yy, xx = np.ogrid[:300, :400]
        for c, (cy, cx, r) in enumerate(((80, 100, 20), (200, 250, 30), (150, 330, 12))):
            im[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0.1 + 0.25 * c
        quiet.append(im)
    imgs = quiet[:2] + busy[:1] + quiet[2:] + busy[1:2]
    want = engine.sift_detect_batch(imgs)
    counts = [want.count(i) for i in range(len(imgs))]
    assert max(counts[:2]) <= 256 < counts[2], counts
    monkeypatch.setenv("PANO_SIFT_CAP", "256")
    eng = Engine(0)
    try:
        got = eng.sift_lazy(imgs, [2, 1, 1, 1])
        _assert_same(got, want, len(imgs))
        pairs = _all_pairs(len(imgs))
        assert _same_matches(eng.match_pairs(got, pairs), engine.match_pairs(want, pairs))
        got.free()
    finally:
        eng.close()
        want.free()


def test_past_the_batch_limit(engine):
    """520 images through one stream: per image the batches of at most 512 images, and matches across image 512
    are those of a featureset uploaded from the downloaded descriptors."""
    from openpano_b200.capi import PanoError
    n = 520
    p = default_params(sift_working_size=200)
    imgs, _ = synth.make_stack(n, 96, 72, 6, 61)
    pix = _pix(imgs)
    batches = [engine.sift_detect_batch_rgb8(pix[:512], p), engine.sift_detect_batch_rgb8(pix[512:], p)]
    with pytest.raises(PanoError):
        engine.sift_detect_batch_rgb8(pix[:513], p)
    pairs = [(510, 511), (511, 512), (512, 513), (505, 515), (0, 519), (300, 517), (518, 519)]
    try:
        for window in ([512, 8], [100] * 5 + [20]):
            got = engine.sift_lazy(pix, window, p)
            try:
                assert got.n_images == n
                _assert_same(got, batches[0], 512)
                _assert_same(got, batches[1], 8, got_at=512)
                descs = [got.download(i)[1] for i in range(n)]
                assert sum(len(d) for d in descs) > 10 * n
                up = engine.featureset_upload(descs)
                want = engine.match_pairs(up, pairs)
                up.free()
                assert sum(len(x) for x in want) > 0
                assert _same_matches(engine.match_pairs(got, pairs), want)
            finally:
                got.free()
    finally:
        for b in batches:
            b.free()


def test_memory_bound(monkeypatch):
    """Over 1 GB of 8-bit sources (12 MP frames, config 5's shape) streamed two at a time: the pool's high-water mark
    stays within one window's SIFT buffers (measured as a batch of two from device sources) plus two windows of
    sources plus twice the packed rows (finish copies them into the featureset's block) plus 64 MB, and below the
    batch path's mark.  Both give the same bits."""
    from openpano_b200.capi import Engine
    monkeypatch.setenv("PANO_CACHE_MB", "0")
    n, W = 30, 2
    imgs, _ = synth.make_stack(n, 4000, 3000, 100, 5)
    pix = _pix(imgs)
    del imgs
    src_u8 = sum(x.nbytes for x in pix)
    assert src_u8 >= 1 << 30
    eng = Engine(0)
    try:
        # one window's SIFT buffers: a batch of W images from device sources, above the sources themselves
        d_pix = [eng.dev_alloc(x.nbytes) for x in pix[:W]]
        for d, x in zip(d_pix, pix):
            eng.dev_upload(d, x)
        eng.sync()
        eng.trim()
        base = eng.mem_high_water(reset=True)
        fs = eng.sift_detect_batch_rgb8_ptr(d_pix, [4000] * W, [3000] * W, [3] * W, device=True)
        fs.count(0)
        eng.sync()
        window_sift = eng.mem_high_water() - base
        fs.free()
        for d in d_pix:
            eng.dev_free(d)
        eng.sync()
        eng.trim()
        eng.mem_high_water(reset=True)

        got = eng.sift_lazy(pix, W)
        eng.sync()
        stream_mark = eng.mem_high_water(reset=True)
        packed = 544 * sum(-(-got.count(i) // 32) * 32 for i in range(n))
        bound = window_sift + 2 * W * pix[0].nbytes + 2 * packed + 64 * MB
        assert stream_mark <= bound, (stream_mark / MB, bound / MB)

        eng.trim()
        eng.mem_high_water(reset=True)
        want = eng.sift_detect_batch_rgb8(pix)
        want.count(0)
        eng.sync()
        batch_mark = eng.mem_high_water()
        _assert_same(got, want, n)
        assert stream_mark < batch_mark - src_u8 // 2, (stream_mark / MB, batch_mark / MB)
        print(f"stream {stream_mark / MB:.0f} MB (bound {bound / MB:.0f} MB: window SIFT {window_sift / MB:.0f}, "
              f"packed {packed / MB:.0f}), batch {batch_mark / MB:.0f} MB, 8-bit sources {src_u8 / MB:.0f} MB")
        got.free()
        want.free()
    finally:
        eng.close()


def test_misuse_is_invalid_and_sticky(engine):
    from openpano_b200.capi import LIB, PanoError, SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_HOST
    imgs, _ = synth.make_stack(4, 240, 180, 60, 71)
    pix = _pix(imgs)
    shapes = [x.shape[:2] for x in pix]
    p = default_params()

    def dims(n):
        return (C.c_int * n)(*[240] * n), (C.c_int * n)(*[180] * n)

    def srcs(k0, k1):
        return (C.c_void_p * max(k1 - k0, 1))(*[pix[k % 4].ctypes.data for k in range(k0, k1)])

    def fresh(n=4):
        h = C.c_void_p()
        ws, hs = dims(n)
        assert LIB.pano_sift_stream_create(engine._h, n, ws, hs, C.byref(p), C.byref(h)) == 0
        return h

    add = LIB.pano_sift_stream_add
    made = []

    def finish(h):
        out = C.c_void_p()
        rc = LIB.pano_sift_stream_finish(h, C.byref(out))
        if out.value:
            made.append(out.value)
        return rc

    cases = {
        "out of order": lambda h: add(h, 1, 1, srcs(1, 2), SRC_RGB8_HOST, 3),
        "overlapping": lambda h: (add(h, 0, 2, srcs(0, 2), SRC_RGB8_HOST, 3), add(h, 1, 1, srcs(1, 2), SRC_RGB8_HOST, 3))[1],
        "excess": lambda h: add(h, 0, 5, srcs(0, 5), SRC_RGB8_HOST, 3),
        "empty": lambda h: add(h, 0, 0, srcs(0, 1), SRC_RGB8_HOST, 3),
        "finish early": lambda h: (add(h, 0, 3, srcs(0, 3), SRC_RGB8_HOST, 3), finish(h))[1],
        "u8 channels": lambda h: add(h, 0, 1, srcs(0, 1), SRC_RGB8_HOST, 2),
        "f32 channels": lambda h: add(h, 0, 1, srcs(0, 1), SRC_F32_HOST, 1),
        "unknown kind": lambda h: add(h, 0, 1, srcs(0, 1), 7, 3),
        "null list": lambda h: add(h, 0, 1, None, SRC_RGB8_HOST, 3),
        "null source": lambda h: add(h, 0, 1, (C.c_void_p * 1)(None), SRC_F32_DEV, 3),
        "null output": lambda h: (add(h, 0, 4, srcs(0, 4), SRC_RGB8_HOST, 3), LIB.pano_sift_stream_finish(h, None))[1],
        "finish twice": lambda h: (add(h, 0, 4, srcs(0, 4), SRC_RGB8_HOST, 3), finish(h), finish(h))[2],
        "add after finish": lambda h: (add(h, 0, 4, srcs(0, 4), SRC_RGB8_HOST, 3), finish(h),
                                       add(h, 4, 1, srcs(0, 1), SRC_RGB8_HOST, 3))[2],
    }
    for name, call in cases.items():
        h = fresh()
        try:
            assert call(h) == -2, name
            assert add(h, 0, 1, srcs(0, 1), SRC_RGB8_HOST, 3) == -2, f"{name}: not sticky"
            assert finish(h) == -2, f"{name}: not sticky"
        finally:
            LIB.pano_sift_stream_free(h)
    # more than one SIFT batch in one add
    h = fresh(600)
    try:
        assert add(h, 0, 513, srcs(0, 513), SRC_RGB8_HOST, 3) == -2
        assert add(h, 0, 512, srcs(0, 512), SRC_RGB8_HOST, 3) == -2, "not sticky"
    finally:
        LIB.pano_sift_stream_free(h)
    for fs in made:                                       # the one successful finish of "finish twice" / "add after finish"
        LIB.pano_featureset_free(fs)
    assert len(made) == 2
    h = C.c_void_p()
    ws, hs = dims(4)
    assert LIB.pano_sift_stream_create(None, 4, ws, hs, C.byref(p), C.byref(h)) == -2
    assert LIB.pano_sift_stream_create(engine._h, 4, ws, hs, C.byref(p), None) == -2
    assert LIB.pano_sift_stream_create(engine._h, 4, None, hs, C.byref(p), C.byref(h)) == -2
    assert LIB.pano_sift_stream_create(engine._h, 0, ws, hs, C.byref(p), C.byref(h)) == -2
    assert LIB.pano_sift_stream_create(engine._h, 4, (C.c_int * 4)(240, 1, 240, 240), hs, C.byref(p), C.byref(h)) == -2
    big_w, big_h = dims(65536)
    assert LIB.pano_sift_stream_create(engine._h, 65536, big_w, big_h, C.byref(p), C.byref(h)) == -2
    assert LIB.pano_sift_stream_add(None, 0, 1, srcs(0, 1), SRC_RGB8_HOST, 3) == -2
    assert LIB.pano_sift_stream_finish(None, None) == -2
    LIB.pano_sift_stream_free(None)
    # the binding checks numpy shapes against the stream's and is sticky as well
    s = engine.sift_stream(shapes)
    try:
        with pytest.raises(PanoError) as ei:
            s.add([pix[0][:-1]])
        assert ei.value.code == -2
        with pytest.raises(PanoError):
            s.add(pix[0:1])
    finally:
        s.close()
    # a stream freed with a window still pending
    s = engine.sift_stream(shapes)
    s.add(pix[0:2])
    s.close()
    # the context is still usable
    want = engine.sift_detect_batch_rgb8(pix)
    got = engine.sift_lazy(pix, 3)
    try:
        _assert_same(got, want, 4)
    finally:
        got.free()
        want.free()


def test_cpp_lazy_detector_equals_reference_detector(tmp_path):
    """B200SIFTDetector::detect_lazy (openpano_b200/host/pano_host.hh) next to the reference's calc_feature loop with
    LAZY_READ (ImageRef::load, SIFTDetector::detect_feature, ImageRef::release) on PPM / PGM files, at windows of
    1, 3 and all images, compiled against the reference's headers (oracle/_ref/lazy_sift_test)."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/lazy_sift_test not built (needs the reference sources at build time)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(tmp_path)], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "LAZY SIFT TEST OK" in out.stdout
    assert out.stdout.count("identical") == 21
