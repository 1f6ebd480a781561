"""GPU: the handle contract of include/pano_b200.h on the four stateful handles (blend stream, SIFT stream, blend
sweep, crop scan), and pano_crop_rect_dev's width limit.  Every misuse returns PANO_ERR_INVALID with its exact
pano_last_error text and launches nothing; every later call on the handle returns the same code and leaves the
message as it is."""
import ctypes as C

import numpy as np
import pytest

from openpano_b200._abi import default_params
from openpano_b200.capi import LIB, PIX_RGBA, SIZE_MAX, SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_DEV, SRC_RGB8_HOST
from tests.test_gpu_blend_strips import _canvas, _gap_stack, _pix

pytestmark = pytest.mark.gpu
INVALID = -2


def _refused(engine, prep, bad, msg, later):
    """prep's calls succeed; bad returns PANO_ERR_INVALID with message msg and launches nothing; then each call of
    later returns it again without a new message."""
    for k, call in enumerate(prep):
        assert call() == 0, (msg, k, LIB.pano_last_error(engine._h).decode())
    launches = engine.launch_count()
    assert bad() == INVALID, msg
    assert LIB.pano_last_error(engine._h).decode() == msg
    assert engine.launch_count() == launches, msg
    for call in later:
        assert call() == INVALID, msg
        assert LIB.pano_last_error(engine._h).decode() == msg


@pytest.fixture(scope="module")
def stack():
    imgs, items, geom = _gap_stack()
    return _pix(imgs), items, geom


@pytest.mark.parametrize("what", ["blend stream", "sift stream"])
def test_stream_misuse(engine, stack, what):
    pix, items, geom = stack
    n = len(pix)
    shapes = [x.shape[:2] for x in pix]
    p = default_params()
    blend = what == "blend stream"
    tw, th = _canvas(items)
    out = np.empty((th, tw, 3), np.float32)
    made = []
    d_rgba = engine.dev_alloc(shapes[0][0] * shapes[0][1] * 4 + 64)

    def create(m=n):
        h = C.c_void_p()
        if blend:
            arr, g = engine._blend_args([None] * n, shapes, items, geom)
            assert LIB.pano_blend_stream_create(engine._h, n, arr, C.byref(g), 0, C.byref(p), tw, th, C.byref(h)) == 0
        else:
            ws = (C.c_int * m)(*[shapes[k % n][1] for k in range(m)])
            hs = (C.c_int * m)(*[shapes[k % n][0] for k in range(m)])
            assert LIB.pano_sift_stream_create(engine._h, m, ws, hs, C.byref(p), C.byref(h)) == 0
        return h

    def srcs(k0, k1):
        return (C.c_void_p * max(k1 - k0, 1))(*[pix[k % n].ctypes.data for k in range(k0, k1)])

    def add(h, first, count, lst, kind=SRC_RGB8_HOST, fmt=3):
        return (LIB.pano_blend_stream_add if blend else LIB.pano_sift_stream_add)(h, first, count, lst, kind, fmt)

    def finish(h, null=False):
        if blend:
            return LIB.pano_blend_stream_finish(h, None if null else out.ctypes.data_as(C.POINTER(C.c_float)))
        fs = C.c_void_p()
        rc = LIB.pano_sift_stream_finish(h, None if null else C.byref(fs))
        if fs.value:
            made.append(fs.value)
        return rc

    free = LIB.pano_blend_stream_free if blend else LIB.pano_sift_stream_free
    cases = [
        ([], lambda h: add(h, 1, 1, srcs(1, 2)), f"{what}: images [1, 2) added, 0 of {n} so far"),
        ([lambda h: add(h, 0, 2, srcs(0, 2))], lambda h: add(h, 1, 1, srcs(1, 2)),
         f"{what}: images [1, 2) added, 2 of {n} so far"),
        ([], lambda h: add(h, 0, n + 1, srcs(0, n + 1)), f"{what}: images [0, {n + 1}) added, 0 of {n} so far"),
        ([], lambda h: add(h, 0, 0, srcs(0, 1)), f"{what}: images [0, 0) added, 0 of {n} so far"),
        ([], lambda h: add(h, -1, 1, srcs(0, 1)), f"{what}: images [-1, 0) added, 0 of {n} so far"),
        ([], lambda h: add(h, 0, 1, None), f"{what}: null source list"),
        ([], lambda h: add(h, 0, 1, (C.c_void_p * 1)(None), SRC_F32_DEV), f"{what}: image 0 has no source"),
        ([lambda h: add(h, 0, 1, srcs(0, 1))], lambda h: add(h, 1, 2, (C.c_void_p * 2)(pix[1].ctypes.data, None)),
         f"{what}: image 2 has no source"),
        ([], lambda h: add(h, 0, 1, srcs(0, 1), 7), f"{what}: unknown source kind 7"),
        ([], lambda h: add(h, 0, 1, None, 7), f"{what}: null source list"),
        ([], lambda h: add(h, 0, 1, srcs(0, 1), SRC_RGB8_HOST, 2), f"{what}: image 0: format 0x2 for source kind 3"),
        ([], lambda h: add(h, 0, 1, srcs(0, 1), SRC_F32_HOST, 1), f"{what}: image 0: format 0x1 for source kind 1"),
        ([], lambda h: add(h, 0, 1, srcs(0, 1), SRC_RGB8_DEV, 0x999),
         f"{what}: image 0: format 0x999 for source kind 2"),
        ([], lambda h: add(h, 0, 1, (C.c_void_p * 1)(d_rgba + 1), SRC_RGB8_DEV, PIX_RGBA),
         f"{what}: image 0: an RGBA source must be 4-byte aligned"),
        ([lambda h: add(h, 0, 3, srcs(0, 3))], lambda h: finish(h), f"{what}: finish after 3 of {n} images"),
        ([lambda h: add(h, 0, n, srcs(0, n))], lambda h: finish(h, null=True), f"{what}: null output"),
        ([lambda h: add(h, 0, n, srcs(0, n)), lambda h: finish(h)], lambda h: finish(h), f"{what}: already finished"),
        ([lambda h: add(h, 0, n, srcs(0, n)), lambda h: finish(h)], lambda h: add(h, n, 1, srcs(0, 1)),
         f"{what}: add after finish"),
        ([lambda h: add(h, 0, n, srcs(0, n)), lambda h: finish(h)], lambda h: add(h, 0, 1, None, 7),
         f"{what}: add after finish"),
    ]
    try:
        for prep, bad, msg in cases:
            h = create()
            try:
                _refused(engine, [lambda c=c: c(h) for c in prep], lambda: bad(h), msg,
                         [lambda: add(h, 0, 1, srcs(0, 1)), lambda: add(h, 0, n, srcs(0, n)), lambda: finish(h)])
            finally:
                free(h)
        if not blend:   # more images in one add than one SIFT batch takes, before the source list is looked at
            for lst in (srcs(0, 513), None):
                h = create(600)
                try:
                    _refused(engine, [], lambda: add(h, 0, 513, lst), "sift stream: 513 images in one add (limit 512)",
                             [lambda: add(h, 0, 512, srcs(0, 512)), lambda: finish(h)])
                finally:
                    free(h)
    finally:
        engine.dev_free(d_rgba)
        for fs in made:
            LIB.pano_featureset_free(fs)
    assert len(made) == (0 if blend else 3)
    assert add(None, 0, 1, srcs(0, 1)) == INVALID and finish(None) == INVALID
    free(None)


def test_row_stream_needed_source(engine, stack):
    """A row stream takes a null source for an image it does not read and refuses one for an image it reads."""
    pix, items, geom = stack
    n = len(pix)
    shapes = [x.shape[:2] for x in pix]
    arr, g = engine._blend_args([None] * n, shapes, items, geom)
    p = default_params()
    tw, th = _canvas(items)
    out = np.empty((40, tw, 3), np.float32)

    def create():
        h = C.c_void_p()
        assert LIB.pano_blend_stream_create_rows(engine._h, n, arr, C.byref(g), 0, C.byref(p), tw, th, 0, 40,
                                                 C.byref(h)) == 0
        return h

    flags = np.zeros(n, np.uint8)
    h = create()
    try:
        assert LIB.pano_blend_stream_needs(h, flags.ctypes.data) == 0
        assert LIB.pano_blend_stream_needs(h, None) == INVALID
        assert LIB.pano_last_error(engine._h).decode() == "blend stream: null flags"
        assert flags[0] == 1 and flags[3] == 0
        read = (C.c_void_p * n)(*[x.ctypes.data if f else None for x, f in zip(pix, flags)])
        assert LIB.pano_blend_stream_add(h, 0, n, read, SRC_RGB8_HOST, 3) == 0
    finally:
        LIB.pano_blend_stream_free(h)
    k = int(np.flatnonzero(flags)[-1])
    lst = (C.c_void_p * n)(*[x.ctypes.data if j != k else None for j, x in enumerate(pix)])
    good = (C.c_void_p * n)(*[x.ctypes.data for x in pix])
    h = create()
    try:
        _refused(engine, [], lambda: LIB.pano_blend_stream_add(h, 0, n, lst, SRC_RGB8_HOST, 3),
                 f"blend stream: image {k} has no source",
                 [lambda: LIB.pano_blend_stream_add(h, 0, n, good, SRC_RGB8_HOST, 3),
                  lambda: LIB.pano_blend_stream_finish(h, out.ctypes.data_as(C.POINTER(C.c_float)))])
    finally:
        LIB.pano_blend_stream_free(h)


def test_sweep_misuse(engine, stack):
    pix, items, geom = stack
    n = len(pix)
    shapes = [x.shape[:2] for x in pix]
    ptrs = [x.ctypes.data for x in pix]
    tw, th = _canvas(items)
    strips = -(-th // 40)
    d_out = engine.dev_alloc(tw * th * 4)
    d_rgba = engine.dev_alloc(max(s[0] * s[1] for s in shapes) * 4 + 64)
    rect = np.zeros(4, np.int32)

    def strip(sw, lst, fmts, kind=SRC_RGB8_HOST):
        src = None if lst is None else (C.c_void_p * n)(*[int(q or 0) for q in lst])
        fm = None if fmts is None else (C.c_int * n)(*fmts)
        return LIB.pano_blend_sweep_strip(sw._h, src, fm, kind)

    def wanted(sw):
        return [q if w else 0 for q, w in zip(ptrs, sw.next()[1])]

    def run_all(sw):
        while sw.next()[0] >= 0:
            if strip(sw, wanted(sw), [3] * n):
                return INVALID
        return 0

    def finish(sw, fmt=3, null=False):
        return LIB.pano_blend_sweep_finish_dev(sw._h, fmt, None if null else C.c_void_p(d_out),
                                               rect.ctypes.data_as(C.POINTER(C.c_int)))

    def first(sw, want=True):
        return int(np.argmax(sw.next()[1] == want))

    def one(sw, k, q, base=None):
        lst = list(base if base is not None else wanted(sw))
        lst[k] = q
        return lst

    def fmts_at(k, f):
        return [f if j == k else 3 for j in range(n)]

    def first_size(sw):
        k = first(sw)
        return k, shapes[k][0] * shapes[k][1]

    cases = [
        ([], lambda sw: strip(sw, None, [3] * n), lambda sw: "blend sweep: null source list"),
        ([], lambda sw: strip(sw, wanted(sw), [3] * n, 7), lambda sw: "blend sweep: unknown source kind 7"),
        ([], lambda sw: strip(sw, None, [3] * n, 7), lambda sw: "blend sweep: null source list"),
        ([], lambda sw: strip(sw, wanted(sw), None), lambda sw: "blend sweep: null format list"),
        ([], lambda sw: strip(sw, one(sw, first(sw), 0), [3] * n),
         lambda sw: f"blend sweep: strip 0 needs image {first(sw)}"),
        ([], lambda sw: strip(sw, one(sw, first(sw, False), ptrs[first(sw, False)]), [3] * n),
         lambda sw: f"blend sweep: strip 0 was not to be given image {first(sw, False)}"),
        ([], lambda sw: strip(sw, wanted(sw), fmts_at(first(sw), 2)),
         lambda sw: f"blend sweep: image {first(sw)}: format 0x2 for source kind 3"),
        ([], lambda sw: strip(sw, [d_rgba + 1 if w else 0 for w in sw.next()[1]], [PIX_RGBA] * n, SRC_RGB8_DEV),
         lambda sw: f"blend sweep: image {first(sw)}: an RGBA source must be 4-byte aligned"),
        ([], lambda sw: strip(sw, wanted(sw), [3] * n, SRC_F32_HOST),
         lambda sw: "blend sweep: image %d takes %d bytes, planned with %d" % (first_size(sw)[0], 12 * first_size(sw)[1],
                                                                               3 * first_size(sw)[1])),
        ([], lambda sw: finish(sw), lambda sw: f"blend sweep: finish after 0 of {strips} strips"),
        ([], lambda sw: finish(sw, null=True), lambda sw: "blend sweep: null output"),
        ([run_all], lambda sw: finish(sw, 1), lambda sw: "blend sweep: output format 0x1"),
        ([run_all], lambda sw: finish(sw, 0x999), lambda sw: "blend sweep: output format 0x999"),
        ([run_all], lambda sw: strip(sw, [0] * n, [3] * n), lambda sw: "blend sweep: strip after the last"),
        ([run_all, finish], lambda sw: finish(sw), lambda sw: "blend sweep: already finished"),
        ([run_all, finish], lambda sw: strip(sw, [0] * n, [3] * n), lambda sw: "blend sweep: strip after the last"),
    ]
    try:
        for prep, bad, msg in cases:
            sw = engine.blend_sweep(shapes, items, geom, 40, SIZE_MAX, 0)
            try:
                text = msg(sw)   # before the refusal: next() still reports the strip's wants
                _refused(engine, [lambda c=c: c(sw) for c in prep], lambda: bad(sw), text,
                         [lambda: strip(sw, [0] * n, [3] * n), lambda: LIB.pano_blend_sweep_next(sw._h, None),
                          lambda: finish(sw)])
            finally:
                sw.close()
    finally:
        engine.dev_free(d_out)
        engine.dev_free(d_rgba)


def test_crop_scan_misuse(engine):
    h = C.c_void_p()
    for w, hh in ((0, 5), (5, 0), (80001, 5), (-1, 5)):
        assert LIB.pano_crop_scan_create(engine._h, w, hh, C.byref(h)) == INVALID
        assert LIB.pano_last_error(engine._h).decode() == f"crop scan: {w}x{hh} (widths 1 to 80000)"
    m = np.zeros((10, 8, 3), np.float32)
    d = engine.dev_alloc(m.nbytes)
    r = np.zeros(4, np.int32)

    def rect(sc, null=False):
        return LIB.pano_crop_scan_rect(sc._h, None if null else r.ctypes.data_as(C.POINTER(C.c_int)))

    def add(sc, ptr, rows):
        return LIB.pano_crop_scan_add_dev(sc._h, C.c_void_p(ptr), rows)

    cases = [
        ([lambda sc: add(sc, d, 6)], lambda sc: add(sc, d, 5), "crop scan: 5 lines at line 6 of 10"),
        ([], lambda sc: add(sc, 0, 3), "crop scan: 3 lines at line 0 of 10"),
        ([], lambda sc: add(sc, d, 0), "crop scan: 0 lines at line 0 of 10"),
        ([], lambda sc: add(sc, d, -1), "crop scan: -1 lines at line 0 of 10"),
        ([lambda sc: add(sc, d, 10)], lambda sc: add(sc, d, 1), "crop scan: 1 lines at line 10 of 10"),
        ([lambda sc: add(sc, d, 4)], lambda sc: rect(sc), "crop scan: rect after 4 of 10 lines"),
        ([lambda sc: add(sc, d, 10)], lambda sc: rect(sc, null=True), "crop scan: null rect"),
    ]
    try:
        engine.dev_upload(d, m)
        for prep, bad, msg in cases:
            sc = engine.crop_scan(8, 10)
            try:
                _refused(engine, [lambda c=c: c(sc) for c in prep], lambda: bad(sc), msg,
                         [lambda: add(sc, d, 1), lambda: rect(sc)])
            finally:
                sc.close()
    finally:
        engine.dev_free(d)
    assert LIB.pano_crop_scan_add_dev(None, None, 1) == INVALID and LIB.pano_crop_scan_rect(None, None) == INVALID
    LIB.pano_crop_scan_free(None)


def test_crop_rect_width_limit(engine):
    """pano_crop_rect_dev takes every width whose line heights fit in shared memory (43,007 columns) and refuses
    wider mosaics with its message."""
    widest = 43007
    d = engine.dev_alloc((widest + 1) * 3 * 4)
    d_rect = engine.dev_alloc(16)
    try:
        engine.dev_upload(d, np.ones((1, widest + 1, 3), np.float32))
        for w in (widest + 1, 80000):
            launches = engine.launch_count()
            assert LIB.pano_crop_rect_dev(engine._h, C.c_void_p(d), w, 1, C.c_void_p(d_rect)) == INVALID
            assert LIB.pano_last_error(engine._h).decode() == \
                f"pano_crop_rect_dev: width {w} exceeds the 40000-column limit"
            assert engine.launch_count() == launches
        for w, hh, ptr in ((0, 1, d), (1, 0, d), (1, 1, 0)):
            assert LIB.pano_crop_rect_dev(engine._h, C.c_void_p(ptr), w, hh, C.c_void_p(d_rect)) == INVALID
            assert LIB.pano_last_error(engine._h).decode() == "pano_crop_rect_dev: bad argument"
        engine.crop_rect_dev(d, widest, 1, d_rect)
        got = np.zeros(4, np.int32)
        engine.dev_download(got, d_rect)
        assert np.array_equal(got, [0, 0, widest, 1])
    finally:
        engine.dev_free(d)
        engine.dev_free(d_rect)
