"""Extrema on the seams of the 64x32 blur tiles.  With the default windows (kw 7 and 13) the
blur kernel tests each tile's interior pixels itself and a second scan tests the tile
perimeters; blobs centred on those seams, in octaves whose last tiles are partial, must give
the oracle's raw, refined and oriented keypoints and descriptors bit for bit.  The generic
windows scan every pixel after the blur and are checked on the same images."""
import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests.test_gpu_sift import compare_trace

pytestmark = pytest.mark.gpu

TILE_W, TILE_H = 64, 32


def _seam_image(w, h, seed):
    """Textured canvas plus bright and dark Gaussian blobs centred on tile seams of octaves 0
    and 1 (working size = input size at these shapes)."""
    rng = np.random.RandomState(seed)
    img = synth.make_canvas(h, w, seed) * np.float32(0.4) + np.float32(0.3)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    w1 = int(np.ceil(np.float32(w) * np.float32(2 ** -0.5)))      # octave-1 width, SCALE_FACTOR sqrt(2)
    to_work = w / w1
    for k in range(160):
        octave = k % 2
        f = 1.0 if octave == 0 else to_work
        sigma = rng.uniform(1.2, 3.0) * f
        if rng.rand() < 0.5:                                       # on a column seam (63 | 64 mod 64)
            cx = (TILE_W * rng.randint(1, int(w / f) // TILE_W + 1) - rng.randint(0, 2)) * f
            cy = rng.uniform(8, h - 8)
        else:                                                      # on a row seam (31 | 32 mod 32)
            cx = rng.uniform(8, w - 8)
            cy = (TILE_H * rng.randint(1, int(h / f) // TILE_H + 1) - rng.randint(0, 2)) * f
        amp = rng.choice([-0.25, 0.25])
        blob = np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / (2 * sigma * sigma)).astype(np.float32)
        img += (amp * blob)[..., None]
    return np.ascontiguousarray(np.clip(img, 0, 1).astype(np.float32))


def _on_seam(pts):
    x, y = pts["x"].astype(np.int64), pts["y"].astype(np.int64)
    return (x % TILE_W == 0) | (x % TILE_W == TILE_W - 1) | (y % TILE_H == 0) | (y % TILE_H == TILE_H - 1)


@pytest.mark.parametrize("w,h,window_factor", [(960, 640, 6), (1000, 600, 6), (960, 640, 4)])
def test_extrema_on_tile_seams(engine, orc, w, h, window_factor):
    img = _seam_image(w, h, 7 + w)
    p = default_params(gauss_window_factor=window_factor)
    g, o = engine.sift_trace(img, p), orc.sift_trace(img, p)
    assert g.working_size() == (w, h)
    raw = o.points(0)
    seam = _on_seam(raw)
    for octave in (0, 1):
        n = int((seam & (raw["pyr_id"] == octave)).sum())
        assert n >= 10, f"octave {octave}: only {n} raw extrema on tile seams"
    w1, h1 = g.octave_size(1)
    assert w1 % TILE_W and h1 % TILE_H, "octave 1 should end in partial tiles"
    assert compare_trace(g, o) > 300
    g.close(); o.close()
