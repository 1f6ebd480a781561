"""CPU: the cylinder sweep's plan (pano_blend_sweep_plan_cyl) and its band rule need no device.  Each strip of the
corrected canvas blends the band of mosaic rows its perspective correction can read: brute force over every output
pixel shows the band holds every row the map reads, for random, keystoned, flipped and all-negative-z corrections;
where z changes sign over a strip the band is the whole mosaic.  The sources are planned over the bands' read sets
as the plain sweep plans them over strips, and the totals match a host recount."""
import numpy as np
import pytest

from openpano_b200.capi import SIZE_MAX, PanoError, blend_sweep_plan_cyl
from tests.persp_util import inv_cases
from tests.test_blend_sweep_plan import _geometry, _reads


def _rows_read(inv, w, h, r0, r1):
    """The mosaic rows the correction of output rows [r0, r1) reads: (min, max) over every pixel, as the kernel
    computes the map (homography.hh:53-64, in double), rounds it to float and floors it (imgproc.cc:135-140); None
    when no tap is read."""
    d = np.asarray(inv, np.float64).reshape(9)
    yy, xx = np.mgrid[r0:r1, 0:w].astype(np.float64)
    rx = d[0] * xx + d[1] * yy + d[2] * 1.0
    ry = d[3] * xx + d[4] * yy + d[5] * 1.0
    rz = d[6] * xx + d[7] * yy + d[8] * 1.0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        denom = 1.0 / rz
        x, y = rx * denom, ry * denom
        ok = (x >= 0) & (x < w) & (y >= 0) & (y < h)
        fr = np.floor(y.astype(np.float32)[ok]).astype(np.int64)
        fc = np.floor(x.astype(np.float32)[ok]).astype(np.int64)
    tap = (fr >= 0) & (fc >= 0) & (fc + 1 < w) & (fr + 1 < h)
    if not tap.any():
        return None
    return int(fr[tap].min()), int(fr[tap].max()) + 1


def _one_image(w, h):
    """A canvas of w×h covered by one image (the plan needs a geometry; the band rule does not read it)."""
    return [(0, 0, w, h, [1.0, 0, 0, 0, 1, 0, 0, 0, 1])], [(h, w)]


@pytest.mark.parametrize("name", ["near", "random", "keystone", "keystone_down", "flip", "negative_z", "z_cross"])
@pytest.mark.parametrize("w,h", [(173, 119), (64, 300)])
def test_band_holds_every_row_read(name, w, h):
    inv = inv_cases(w, h, seed=w)[name]
    items, shapes = _one_image(w, h)
    geom = {"projection": 0, "res_x": 1.0, "res_y": 1.0, "proj_min_x": 0.0, "proj_min_y": 0.0}
    for rows in (1, 7, 21, h // 2, h):
        pl = blend_sweep_plan_cyl(shapes, items, geom, 0, inv, rows, [w * h * 3], SIZE_MAX)
        for s, (b0, b1) in enumerate(pl["band"]):
            r0, r1 = s * rows, min(h, (s + 1) * rows)
            assert 0 <= b0 <= b1 <= h
            d = inv.reshape(9)
            z = [d[6] * x + d[7] * y + d[8] for x in (0, w - 1) for y in (r0, r1 - 1)]
            if min(z) <= 0 <= max(z):
                assert (b0, b1) == (0, h), (name, rows, s)               # z changes sign: the whole mosaic
            got = _rows_read(inv, w, h, r0, r1)
            if got is not None:
                assert b0 <= got[0] and got[1] < b1, (name, rows, s, got, (b0, b1))
            assert pl["reads"][s].any() == (b0 < b1), (name, rows, s)
    if name == "keystone":           # a strongly keystoned correction reads bands much taller than its strips
        pl = blend_sweep_plan_cyl(shapes, items, geom, 0, inv, 1, [w * h * 3], SIZE_MAX)
        assert (pl["band"][:, 1] - pl["band"][:, 0]).max() >= 4


def _plan_over(reads, nbytes, keep):
    """The farthest-next-use schedule over given per-strip read sets (test_blend_sweep_plan's restatement)."""
    S, n = reads.shape
    nxt = np.full((S, n), S)
    for s in range(S - 2, -1, -1):
        nxt[s] = np.where(reads[s + 1], s + 1, nxt[s + 1])
    uploads, kept = np.zeros((S, n), bool), np.zeros((S, n), bool)
    resident, high = set(), 0
    for s in range(S):
        uploads[s] = reads[s] & ~np.isin(np.arange(n), list(resident))
        cand = [k for k in range(n) if (k in resident or reads[s, k]) and nxt[s, k] < S]
        cand.sort(key=lambda k: (-nxt[s, k], -k))
        total, q = sum(nbytes[k] for k in cand), 0
        while q < len(cand) and total > keep:
            total -= nbytes[cand[q]]
            q += 1
        resident = set(cand[q:])
        kept[s] = uploads[s] & np.isin(np.arange(n), list(resident))
        high = max(high, total)
    return uploads, kept, high


@pytest.mark.parametrize("bands", [0, 2, 5])
@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("name", ["near", "keystone", "flip", "z_cross"])
def test_plan_reads_the_bands(bands, seed, name):
    items, shapes, geom = _geometry(seed * 10, 0)
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    inv = inv_cases(ow, oh, seed)[name]
    nbytes = [h * w * (1 + (k % 4)) for k, (h, w) in enumerate(shapes)]
    for rows in (1, 21, 256, oh):
        for keep in (0, max(nbytes), sum(nbytes) // 3, SIZE_MAX):
            pl = blend_sweep_plan_cyl(shapes, items, geom, bands, inv, rows, nbytes, keep)
            reads = np.array([_reads(items, bands, b0, b1, oh) if b0 < b1 else np.zeros(len(items), bool)
                              for b0, b1 in pl["band"]])
            key = (rows, keep)
            assert np.array_equal(pl["reads"], reads), key
            uploads, kept, high = _plan_over(reads, nbytes, keep)
            assert np.array_equal(pl["uploads"], uploads), key
            assert np.array_equal(pl["kept"], kept), key
            assert pl["retained_high"] == high <= keep, key
            assert pl["n_uploads"] == uploads.sum(), key
            assert pl["upload_bytes"] == sum(int(nbytes[k]) * int(c) for k, c in enumerate(uploads.sum(0))), key
            if keep == SIZE_MAX:                                   # each read source handed over exactly once
                assert np.array_equal(pl["uploads"].sum(0), reads.any(0).astype(int)), key
            if keep == 0:
                assert np.array_equal(pl["uploads"], reads) and not pl["kept"].any(), key


def test_plan_rejects_bad_arguments():
    items, shapes, geom = _geometry(3, 0)
    nbytes = [1] * len(items)
    inv = np.eye(3)
    for rows, nb in ((0, nbytes), (5, [0] * len(items))):
        with pytest.raises(PanoError):
            blend_sweep_plan_cyl(shapes, items, geom, 0, inv, rows, nb, 0)
    from openpano_b200 import capi
    arr, g = capi.Engine._blend_args([None] * len(items), shapes, items, geom)
    p = capi.default_params()
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    nb = (capi.C.c_size_t * len(items))(*nbytes)
    assert capi.LIB.pano_blend_sweep_plan_cyl(len(items), arr, capi.C.byref(g), 0, capi.C.byref(p), ow, oh, None, 5,
                                              nb, 0, None, None, None, None, None, None, None, None) == -2
