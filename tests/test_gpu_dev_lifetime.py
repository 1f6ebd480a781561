"""GPU: with PANO_CACHE_MB=0 (no block cache, no kept SIFT plan) every entry point gives back every pool block it
took, on success and on a failure after its inputs were validated: after each call the pool holds only the
caller's buffers again.  And a context gives back its pinned host memory, events and streams when it closes."""
import ctypes

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200.capi import LIB, SRC_F32_DEV, PanoError
from openpano_b200._abi import default_params
from tests.ba_util import ba_case, numpy_pair_mats
from tests.ransac_util import ransac_case

pytestmark = pytest.mark.gpu

W, H, N = 320, 240, 3


def _in_use(e):
    e.sync()
    e.mem_high_water(reset=True)       # the mark restarts at what is in use now
    return e.mem_high_water()


@pytest.fixture
def eng(monkeypatch):
    from openpano_b200.capi import Engine
    monkeypatch.setenv("PANO_CACHE_MB", "0")
    e = Engine(0)
    yield e
    e.close()


def test_every_entry_point_gives_its_blocks_back(eng):
    p = default_params()
    imgs, org = synth.make_stack(N, W, H, 120, 3)
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    items, geom = synth.translation_blend_setup(org, W, H)
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)

    # descriptor sets to upload and import (SIFT keeps nothing here: no cache, no plan)
    fs = eng.sift_detect_batch(imgs, p)
    descs, coors = zip(*[fs.download(i)[::-1] for i in range(N)])
    fs.free()
    counts = [len(d) for d in descs]

    # the caller's buffers first, then the planet table (it lives as long as the context)
    d_img = [eng.dev_alloc(im.nbytes) for im in imgs]
    d_pix = [eng.dev_alloc(x.nbytes) for x in pix]
    for d, x in zip(d_img + d_pix, imgs + pix):
        eng.dev_upload(d, np.ascontiguousarray(x))
    d_out = eng.dev_alloc(ow * oh * 3 * 4)
    wshape = [eng.cyl_warp_shape(W, H, 1.0, p)[:2] for _ in range(N)]
    d_warp = [eng.dev_alloc(w * h * 3 * 4) for w, h in wshape]
    d_planet = eng.dev_alloc(1000 * 1000 * 3 * 4)
    d_rect = eng.dev_alloc(256)
    d_rgb8 = eng.dev_alloc(ow * oh * 3)
    d_desc = eng.dev_alloc(max(sum(counts), 1) * 128 * 4)
    d_coor = eng.dev_alloc(max(sum(counts), 1) * 2 * 8)
    eng.planet_dev(d_img[0], W, H, d_planet)
    base = _in_use(eng)

    def cycle(what, fn):
        fn()
        assert _in_use(eng) == base, what

    def fails(fn):
        with pytest.raises(PanoError):
            fn()

    # SIFT: f32 and 8-bit sources, host and device
    def sift(fs):
        [fs.count(i) for i in range(N)]
        fs.free()

    chans = [3] * N
    cycle("sift f32 host", lambda: sift(eng.sift_detect_batch(imgs, p)))
    cycle("sift f32 dev", lambda: sift(eng.sift_detect_batch_ptr(d_img, [W] * N, [H] * N, p, device=True)))
    cycle("sift rgb8 host", lambda: sift(eng.sift_detect_batch_rgb8(pix, p)))
    cycle("sift rgb8 dev", lambda: sift(eng.sift_detect_batch_rgb8_ptr(d_pix, [W] * N, [H] * N, chans, p, device=True)))
    cycle("sift trace", lambda: eng.sift_trace(imgs[0], p).close())

    # featuresets: upload and device import, each matched (sharded and not), plus a pair index out of range
    off = 0
    d_descs, d_coors = [], []
    for d, c in zip(descs, coors):
        eng.dev_upload(d_desc + off * 128 * 4, np.ascontiguousarray(d, np.float32))
        eng.dev_upload(d_coor + off * 2 * 8, np.ascontiguousarray(c, np.float64))
        d_descs.append(d_desc + off * 128 * 4)
        d_coors.append(d_coor + off * 2 * 8)
        off += len(d)
    assert _in_use(eng) == base
    pairs = [(0, 1), (1, 2), (0, 2)]

    def match(fs):
        try:
            eng.match_pairs(fs, pairs, p)
            eng.match_pairs(fs, pairs, p, shard=(1, 2))
            eng.match_pairs_dev(fs, pairs, p)
            eng.match_pairs_dev(fs, pairs, p, shard=(0, 2))
            fails(lambda: eng.match_pairs(fs, [(0, N)], p))
            fails(lambda: eng.match_pairs_dev(fs, [(0, N)], p))
        finally:
            fs.free()

    cycle("featureset upload + match", lambda: match(eng.featureset_upload(descs, coors)))
    cycle("featureset import + match", lambda: match(eng.featureset_import_dev(counts, d_descs, d_coors)))

    # RANSAC scoring, the one-shot BA Jacobian and a BA session
    cycle("ransac", lambda: eng.ransac_score_pairs([ransac_case(200, 64, 5), ransac_case(80, 16, 6)]))
    cams, bpairs, bpts = ba_case(5, 40, 5, extra_pairs=3)
    mats = numpy_pair_mats(cams, bpairs)
    cycle("ba jacobian", lambda: eng.ba_jacobian(5, [(f, t, n, m) for (f, t, n), m in zip(bpairs, mats)], bpts[:, :2]))

    def ba_session():
        s = eng.ba_session(5, bpairs, bpts)
        try:
            s.error(np.tile(np.eye(3).reshape(-1), (len(bpairs), 1)))
            s.normal_equations(mats, want_rows=True)
        finally:
            s.close()

    cycle("ba session", ba_session)

    # cylinder warps: host, and both device batches
    cycle("cyl_warp", lambda: eng.cyl_warp(imgs[0], None, 1.0, p))
    shapes = [(H, W)] * N
    cycle("cyl_warp_batch", lambda: eng.cyl_warp_batch_dev(d_img, shapes, d_warp, None, 1.0, p))
    cycle("cyl_warp_batch rgb8", lambda: eng.cyl_warp_batch_rgb8_dev(d_pix, chans, shapes, d_warp, None, 1.0, p))

    # blends, linear and multiband
    for bands in (0, 3):
        cycle(f"blend {bands}", lambda: eng.blend(imgs, items, geom, bands, p))
        cycle(f"blend_dev {bands}", lambda: eng.blend_dev(d_img, shapes, items, geom, d_out, ow, oh, bands, p))
        cycle(f"blend_rgb8_dev {bands}",
              lambda: eng.blend_rgb8_dev(d_pix, chans, shapes, items, geom, d_out, ow, oh, bands, p))
        cycle(f"blend_rows_dev {bands}",
              lambda: eng.blend_rows_dev(d_img, shapes, items, geom, d_out, ow, oh, oh // 3, oh // 2, bands, p))
        cycle(f"blend_rows_rgb8_dev {bands}",
              lambda: eng.blend_rows_rgb8_dev(d_pix, chans, shapes, items, geom, d_out, ow, oh, oh // 3, oh // 2, bands,
                                              p))
        # a strip no image reaches: every image below it
        low = [(x0, y0 + oh, x1, y1 + oh, hi) for x0, y0, x1, y1, hi in items]
        cycle(f"blend_rows_dev empty strip {bands}",
              lambda: eng.blend_rows_dev(d_img, shapes, low, geom, d_out, ow, 2 * oh, 0, oh // 2, bands, p))

        # blend streams: one finished, one closed before it finishes, one refused an add out of order
        def stream_finished():
            s = eng.blend_stream(shapes, items, geom, bands, p)
            try:
                s.add(imgs[:2])
                s.add(pix[2:])
                s.finish()
            finally:
                s.close()

        def stream_closed():
            s = eng.blend_stream(shapes, items, geom, bands, p)
            try:
                s.add(imgs[:1])
            finally:
                s.close()

        def stream_misused():
            s = eng.blend_stream(shapes, items, geom, bands, p)
            try:
                s.add(imgs[:1])
                # image 1 comes next: adding image 2 is refused
                assert LIB.pano_blend_stream_add(s._h, 2, 1, (ctypes.c_void_p * 1)(d_img[2]), SRC_F32_DEV, 3) != 0
            finally:
                s.close()

        cycle(f"blend stream finished {bands}", stream_finished)
        cycle(f"blend stream closed {bands}", stream_closed)
        cycle(f"blend stream add out of order {bands}", stream_misused)

    # little planet, the image-I/O conversions and the crop rectangle
    cycle("planet", lambda: eng.planet(imgs[0]))
    cycle("read_img", lambda: eng.read_img_rgb8(pix[0]))
    cycle("rgb8_to_mat32f_batch", lambda: eng.rgb8_to_mat32f_batch_dev(d_pix, [W] * N, [H] * N, chans, d_img))
    cycle("crop_rect", lambda: eng.crop_rect_dev(d_out, ow, oh, d_rect))
    cycle("mat32f_to_rgb8", lambda: eng.mat32f_to_rgb8_dev(d_out, ow, oh, d_rect, d_rgb8))
    cycle("crop_write_rgb8", lambda: eng.crop_write_rgb8(imgs[1]))

    for d in d_img + d_pix + d_warp + [d_out, d_planet, d_rect, d_rgb8, d_desc, d_coor]:
        eng.dev_free(d)


def _rss_bytes():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) * 1024
    raise AssertionError("no VmRSS in /proc/self/status")


def test_closed_contexts_give_their_host_resources_back():
    """Each cycle opens a context, takes every pinned-memory and event path once and closes it.  Pinned pages count
    in the process's resident set, and one context holds at least its 8 MB ring, so contexts that kept their pinned
    memory would grow it by that much per cycle."""
    from openpano_b200.capi import Engine
    p = default_params()
    imgs, org = synth.make_stack(N, W, H, 120, 3)
    items, geom = synth.translation_blend_setup(org, W, H)
    shapes = [(H, W)] * N
    pairs = [(0, 1), (1, 2), (0, 2)]
    rcases = [ransac_case(200, 64, 5), ransac_case(80, 16, 6)]
    cams, bpairs, bpts = ba_case(5, 40, 5, extra_pairs=3)
    hto = np.tile(np.eye(3).reshape(-1), (len(bpairs), 1))

    def cycle():
        e = Engine(0)
        try:
            fs = e.sift_detect_batch(imgs, p)              # pageable sources: staging buffer A
            try:
                e.match_pairs(fs, pairs, p)                # the mapped ring and the completion-marker word
            finally:
                fs.free()
            e.ransac_score_pairs(rcases)                   # staging buffers A and B
            s = e.ba_session(5, bpairs, bpts)              # a recycled mapped block; B for the residuals
            try:
                s.error(hto, want_residuals=True)
            finally:
                s.close()
            bs = e.blend_stream(shapes, items, geom, 0, p)  # its copy stream, events and pinned staging
            try:
                bs.add(imgs[:2])
                bs.add(imgs[2:])
                bs.finish()
            finally:
                bs.close()
            e.profile(True)                                # pooled timing events
            e.ransac_score_pairs(rcases)
            e.profile(False)
            ev = e.event_create()
            e.event_record(ev)
            Engine.event_sync(ev)
            Engine.event_destroy(ev)
        finally:
            e.close()

    cycles, ring_bytes = 20, 8 << 20
    for _ in range(2):          # first-use costs of the driver, the library and the allocator
        cycle()
    rss0 = _rss_bytes()
    for _ in range(cycles):
        cycle()
    grown = _rss_bytes() - rss0
    assert grown < cycles * ring_bytes // 4, f"resident set grew by {grown / 2**20:.1f} MB over {cycles} contexts"
