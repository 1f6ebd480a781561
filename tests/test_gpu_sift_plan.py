"""GPU: a context keeps the last SIFT batch's shape-dependent setup (its plan) and reuses it for a batch of the same
shapes.  Every batch must give the features a fresh context gives (PANO_CACHE_MB=0 keeps no plan), bit for bit:
repeats, new images at new device addresses, changed shapes / n / params, f32 after 8-bit sources and a capacity
retry.  With PANO_CACHE_MB=0 nothing stays allocated after a batch, and pano_trim gives the plan back to the
pool."""
import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params

pytestmark = pytest.mark.gpu

SHAPES = [(600, 400), (640, 480), (333, 517)]


def _imgs(shapes, seed):
    return [synth.make_canvas(h, w, seed + 7 * k) for k, (w, h) in enumerate(shapes)]


def _pix(imgs):
    return [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]


class Batch:
    """Device copies of a batch's sources on one engine."""

    def __init__(self, eng, srcs):
        self.eng, self.srcs = eng, srcs
        self.ptrs = [eng.dev_alloc(x.nbytes) for x in srcs]
        for d, x in zip(self.ptrs, srcs):
            eng.dev_upload(d, np.ascontiguousarray(x))

    def sift(self, p):
        ws, hs = [x.shape[1] for x in self.srcs], [x.shape[0] for x in self.srcs]
        if self.srcs[0].dtype == np.uint8:
            chans = [1 if x.ndim == 2 else 3 for x in self.srcs]
            fs = self.eng.sift_detect_batch_rgb8_ptr(self.ptrs, ws, hs, chans, p, device=True)
        else:
            fs = self.eng.sift_detect_batch_ptr(self.ptrs, ws, hs, p, device=True)
        try:
            return [fs.download(i) for i in range(len(self.srcs))]
        finally:
            fs.free()

    def free(self):
        for d in self.ptrs:
            self.eng.dev_free(d)


def _fresh(monkeypatch, srcs, p):
    """The features of a context that keeps no plan."""
    from openpano_b200.capi import Engine
    with monkeypatch.context() as m:
        m.setenv("PANO_CACHE_MB", "0")
        eng = Engine(0)
    try:
        b = Batch(eng, srcs)
        got = b.sift(p)
        b.free()
        return got
    finally:
        eng.close()


def _same(got, want):
    assert len(got) == len(want)
    for i, ((c, d), (co, do)) in enumerate(zip(got, want)):
        assert c.shape == co.shape and d.shape == do.shape, i
        assert c.tobytes() == co.tobytes() and d.tobytes() == do.tobytes(), i


@pytest.fixture
def eng(monkeypatch):
    from openpano_b200.capi import Engine
    monkeypatch.delenv("PANO_CACHE_MB", raising=False)
    e = Engine(0)
    yield e
    e.close()


def test_repeat_and_new_images(monkeypatch, eng):
    """The same shapes twice, then other images of the same shapes at other device addresses, then the first
    images again."""
    p = default_params()
    a_src, b_src = _imgs(SHAPES, 11), _imgs(SHAPES, 12)
    want_a, want_b = _fresh(monkeypatch, a_src, p), _fresh(monkeypatch, b_src, p)
    assert min(len(d) for _, d in want_a) > 100
    a, b = Batch(eng, a_src), Batch(eng, b_src)
    try:
        for batch, want in ((a, want_a), (a, want_a), (b, want_b), (a, want_a), (b, want_b)):
            _same(batch.sift(p), want)
    finally:
        a.free()
        b.free()


def test_shapes_n_and_params_change(monkeypatch, eng):
    p, p5 = default_params(), default_params(num_octave=5, scale_factor=1.3)
    # same shapes, other tables: the Gaussian taps, the orientation smoothing and the descriptor scale
    pg, po, pd = default_params(gauss_sigma=1.6), default_params(ori_hist_smooth_count=0), default_params(desc_int_factor=100)
    full, other = _imgs(SHAPES, 21), _imgs([(517, 333), (800, 600), (641, 417)], 22)
    cases = [(full, p), (full[:2], p), (other, p), (full, p5), (full, p), (full[1:], p5), (full, p),
             (full, pg), (full, po), (full, pd), (full, p)]
    for srcs, params in cases:
        b = Batch(eng, srcs)
        try:
            _same(b.sift(params), _fresh(monkeypatch, srcs, params))
        finally:
            b.free()


def test_f32_then_rgb8_sources(monkeypatch, eng):
    """One shape list read as 8-bit RGB, as f32 (read_img's conversion of the same pixels, hence the same
    features), as 8-bit grey, and as 8-bit RGB again."""
    p = default_params()
    pix = _pix(_imgs(SHAPES, 31))
    f32 = [(x.astype(np.float32).astype(np.float64) / 255.0).astype(np.float32) for x in pix]
    grey = [np.ascontiguousarray(x[..., 1]) for x in pix]
    want_rgb, want_grey = _fresh(monkeypatch, pix, p), _fresh(monkeypatch, grey, p)
    _same(_fresh(monkeypatch, f32, p), want_rgb)
    for srcs, want in ((f32, want_rgb), (pix, want_rgb), (grey, want_grey), (f32, want_rgb), (pix, want_rgb)):
        b = Batch(eng, srcs)
        try:
            _same(b.sift(p), want)
        finally:
            b.free()


def test_capacity_retry_then_repeat(monkeypatch):
    """Lists that start at 256 entries overflow: the batch runs again with larger lists (a new plan), and the
    next batch of the same shapes starts at the grown capacity."""
    from openpano_b200.capi import Engine
    p = default_params()
    srcs = _imgs([(1300, 867), (600, 400)], 41)
    want = _fresh(monkeypatch, srcs, p)
    assert max(len(d) for _, d in want) > 256
    monkeypatch.delenv("PANO_CACHE_MB", raising=False)
    monkeypatch.setenv("PANO_SIFT_CAP", "256")
    e = Engine(0)
    try:
        b = Batch(e, srcs)
        for _ in range(3):
            _same(b.sift(p), want)
        b.free()
    finally:
        e.close()


def _in_use(e):
    e.sync()
    e.mem_high_water(reset=True)       # the mark restarts at what is in use now
    return e.mem_high_water()


def test_cache_off_keeps_no_plan(monkeypatch):
    """PANO_CACHE_MB=0: after fs.free() the pool holds only the caller's buffers, and every batch of the same
    shapes reaches the same high-water mark."""
    from openpano_b200.capi import Engine
    monkeypatch.setenv("PANO_CACHE_MB", "0")
    e = Engine(0)
    try:
        b = Batch(e, _imgs(SHAPES, 61))
        base = _in_use(e)
        marks = []
        for _ in range(3):
            b.sift(default_params())
            e.sync()
            marks.append(e.mem_high_water(reset=True))
            assert e.mem_high_water() == base
        assert marks[0] > base and marks[0] == marks[1] == marks[2], marks
        b.free()
    finally:
        e.close()


def test_trim_releases_plan(eng):
    b = Batch(eng, _imgs(SHAPES, 71))
    try:
        base = _in_use(eng)
        b.sift(default_params())
        assert _in_use(eng) > base            # the plan (and the cache) hold blocks
        eng.trim()
        assert _in_use(eng) == base
        b.sift(default_params())              # a trimmed context builds its plan again
    finally:
        b.free()
