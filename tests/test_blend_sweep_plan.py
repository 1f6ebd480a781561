"""CPU: pano_blend_sweep_plan, the strip schedule of a blend sweep, needs no device.  It is compared with a plain
restatement of the strip read rule (pano_blend_stream_needs) and of the farthest-next-use policy on seeded random
geometries, and checked for the properties its header states: keep_bytes 0 hands over every read of every strip,
an unlimited budget each read image once, the kept bytes never exceed the budget, and an image no strip reads is
never asked for."""
import numpy as np
import pytest

from openpano_b200.capi import SIZE_MAX, PanoError, blend_sweep_plan

# summed blur half-widths of the multiband levels at GAUSS_WINDOW_FACTOR 6 (include/pano_b200.h)
HALO = {0: 0, 1: 0, 2: 6, 5: 27}


def _reads(items, bands, r0, r1, oh):
    if r0 == 0 and r1 == oh:
        return np.ones(len(items), bool)
    if bands == 0:
        return np.array([y0 < r1 and y1 >= r0 for _, y0, _, y1, _ in items])
    c0 = max(0, r0 - HALO[bands]) if r0 > 0 else -(1 << 40)
    c1 = r1 + HALO[bands] - 1 if r1 < oh else 1 << 40
    return np.array([max(y0, c0) <= min(y1, c1) for _, y0, _, y1, _ in items])


def _plan(items, bands, rows, nbytes, keep):
    n, oh = len(items), max(it[3] for it in items)
    S = -(-oh // rows)
    reads = np.array([_reads(items, bands, s * rows, min(oh, (s + 1) * rows), oh) for s in range(S)])
    nxt = np.full((S, n), S)
    for s in range(S - 2, -1, -1):
        nxt[s] = np.where(reads[s + 1], s + 1, nxt[s + 1])
    uploads, kept = np.zeros((S, n), bool), np.zeros((S, n), bool)
    resident, high = set(), 0
    for s in range(S):
        uploads[s] = reads[s] & ~np.isin(np.arange(n), list(resident))
        cand = [k for k in range(n) if (k in resident or reads[s, k]) and nxt[s, k] < S]
        cand.sort(key=lambda k: (-nxt[s, k], -k))          # the farthest next use goes first, then the higher index
        total, q = sum(nbytes[k] for k in cand), 0
        while q < len(cand) and total > keep:
            total -= nbytes[cand[q]]
            q += 1
        resident = set(cand[q:])
        kept[s] = uploads[s] & np.isin(np.arange(n), list(resident))
        high = max(high, total)
    return reads, uploads, kept, high


def _geometry(seed, projection):
    rng = np.random.RandomState(seed)
    n = int(rng.randint(3, 14))
    W, H = int(rng.randint(200, 900)), int(rng.randint(120, 500))
    items, shapes = [], []
    for _ in range(n):
        w, h = int(rng.randint(20, W // 2)), int(rng.randint(10, H // 2))
        x0, y0 = int(rng.randint(0, W - w)), int(rng.randint(0, H - h))
        items.append((x0, y0, x0 + w, y0 + h, list(rng.standard_normal(9))))
        shapes.append((int(rng.randint(2, 300)), int(rng.randint(2, 300))))
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    items.append((0, oh, ow, oh, [1.0, 0, 0, 0, 1, 0, 0, 0, 1]))       # one row at the bottom edge
    shapes.append((5, 5))
    geom = {"projection": projection, "res_x": 0.01, "res_y": 0.01, "proj_min_x": -1.0, "proj_min_y": -0.5}
    return items, shapes, geom


@pytest.mark.parametrize("projection", [0, 1, 2])
@pytest.mark.parametrize("bands", [0, 1, 2, 5])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_plan_equals_restatement(projection, bands, seed):
    items, shapes, geom = _geometry(seed * 10 + projection, projection)
    oh = max(it[3] for it in items)
    nbytes = [h * w * (1 + (k % 4)) for k, (h, w) in enumerate(shapes)]
    for rows in (1, 7, oh, oh + 5):
        for keep in (0, max(nbytes), sum(nbytes) // 3, SIZE_MAX):
            pl = blend_sweep_plan(shapes, items, geom, bands, rows, nbytes, keep)
            reads, uploads, kept, high = _plan(items, bands, rows, nbytes, keep)
            key = (rows, keep)
            assert np.array_equal(pl["reads"], reads), key
            assert np.array_equal(pl["uploads"], uploads), key
            assert np.array_equal(pl["kept"], kept), key
            assert pl["retained_high"] == high, key
            assert pl["n_uploads"] == uploads.sum(), key
            assert pl["upload_bytes"] == sum(int(nbytes[k]) * int(c) for k, c in enumerate(uploads.sum(0))), key
            assert pl["retained_high"] <= keep
            read_any = reads.any(0)
            assert not uploads[:, ~read_any].any(), key                 # never asked for an image no strip reads
            assert (uploads <= reads).all()
            if keep == 0:
                assert np.array_equal(uploads, reads) and not kept.any()
            if keep == SIZE_MAX:
                assert np.array_equal(uploads.sum(0), read_any.astype(int)), key


def test_plan_strip_heights_and_totals():
    items, shapes, geom = _geometry(7, 0)
    oh = max(it[3] for it in items)
    nbytes = [h * w * 3 for h, w in shapes]
    assert blend_sweep_plan(shapes, items, geom, 0, 1, nbytes, 0)["reads"].shape == (oh, len(items))
    for rows in (oh, oh + 1, 10 * oh):
        pl = blend_sweep_plan(shapes, items, geom, 5, rows, nbytes, 0)
        assert pl["reads"].shape == (1, len(items)) and pl["reads"].all()       # one strip: the whole canvas


def test_plan_config5_traffic():
    """Config 5's blend: 64 frames of 4000×3000 on a grid in an 8000×6000 canvas, 8-bit RGB.  At strips of 256 rows
    an unlimited budget hands over the sources' 2.3 GB once, against 14 GB without keeping any."""
    w, h = 4000, 3000
    org = [(c * 4000 // 7, r * 3000 // 7) for r in range(8) for c in range(8)]
    items = [(x, y, x + w - 1, y + h - 1, [1.0, 0, -x, 0, 1, -y, 0, 0, 1]) for x, y in org]
    shapes = [(h, w)] * 64
    geom = {"projection": 0, "res_x": 1.0, "res_y": 1.0, "proj_min_x": 0.0, "proj_min_y": 0.0}
    nbytes = [w * h * 3] * 64
    once = blend_sweep_plan(shapes, items, geom, 0, 256, nbytes, SIZE_MAX)
    none = blend_sweep_plan(shapes, items, geom, 0, 256, nbytes, 0)
    assert once["upload_bytes"] == 64 * w * h * 3
    assert none["upload_bytes"] > 5 * once["upload_bytes"]
    assert once["retained_high"] < once["upload_bytes"]


def test_plan_rejects_bad_arguments():
    items, shapes, geom = _geometry(3, 0)
    nbytes = [1] * len(items)
    for rows, nb in ((0, nbytes), (5, [0] * len(items))):
        with pytest.raises(PanoError):
            blend_sweep_plan(shapes, items, geom, 0, rows, nb, 0)
    with pytest.raises(PanoError):
        blend_sweep_plan([(1, 5)] + shapes[1:], items, geom, 0, 5, nbytes, 0)
