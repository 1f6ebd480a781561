"""Checker wrappers and cases for cylinder mode's perspective correction, CylinderStitcher::perspective_correction
(cylstitcher.cc:139-180): orc_persp_correct (the plain-C restatement, oracle/liboracle_persp.so) and
ref_persp_correction (the reference's own pass, oracle/_ref/libopenpano_ref_persp.so), both built by
oracle/cyl_sweep.mk."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ORC_SO = ROOT / "oracle" / "liboracle_persp.so"
REF_SO = ROOT / "oracle" / "_ref" / "libopenpano_ref_persp.so"
_libs = {}


def _lib(path):
    if path not in _libs:
        if path == ORC_SO and not path.exists():
            subprocess.check_call(["make", "-s", "-C", str(ROOT / "oracle"), "-f", "cyl_sweep.mk", "oracle"])
        _libs[path] = C.CDLL(str(path))
    return _libs[path]


def have_ref():
    return REF_SO.exists()


def _correct(fn, mosaic, inv, lazy, ordered):
    m = np.ascontiguousarray(mosaic, np.float32)
    h, w = m.shape[:2]
    d = np.ascontiguousarray(np.asarray(inv, np.float64).reshape(9))
    out = np.empty_like(m)
    rc = fn(C.c_void_p(m.ctypes.data), w, h, C.c_void_p(d.ctypes.data), int(lazy), int(ordered),
            C.c_void_p(out.ctypes.data))
    assert rc == 0
    return out


def orc_correct(mosaic, inv, lazy=1, ordered=1):
    """The plain-C correction pass of an h×w×3 f32 mosaic (LAZY_READ lazy, ORDERED_INPUT ordered)."""
    return _correct(_lib(ORC_SO).orc_persp_correct, mosaic, inv, lazy, ordered)


def ref_correct(mosaic, inv, lazy=1, ordered=1):
    """The reference's perspective_correction of the mosaic with its correction homography handed over as inv."""
    return _correct(_lib(REF_SO).ref_persp_correction, mosaic, inv, lazy, ordered)


def keystone(w, h, top=0.3, bottom=0.0, shift=0.0):
    """inv of getPerspectiveTransform's kind for a w×h canvas: the corrected rectangle's corners (0, 0), (0, h),
    (w, 0), (w, h) map to a trapezoid of the mosaic whose top edge is `top` · w narrower than the bottom one (and
    the bottom edge `bottom` · w), moved down by shift · h.  Solved in double with numpy (the engine takes inv as
    given)."""
    src = [(0, 0), (0, h), (w, 0), (w, h)]
    dst = [(top * w / 2, shift * h), (bottom * w / 2, h * (1 - 0.1 * abs(shift)) + shift * h),
           (w - top * w / 2, shift * h), (w - bottom * w / 2, h * (1 - 0.1 * abs(shift)) + shift * h)]
    A, b = [], []
    for (x, y), (u, v) in zip(src, dst):
        A.append([x, y, 1, 0, 0, 0, -u * x, -u * y]); b.append(u)
        A.append([0, 0, 0, x, y, 1, -v * x, -v * y]); b.append(v)
    sol = np.linalg.solve(np.array(A, np.float64), np.array(b, np.float64))
    return np.append(sol, 1.0).reshape(3, 3)


def inv_cases(w, h, seed=0):
    """name -> inv: near identity, a random small projective, strongly keystoned, flipped, all-negative z (the same
    map, every z below 0), and a z that changes sign across the canvas."""
    rng = np.random.RandomState(seed)
    near = np.eye(3) + np.diag([0.01, -0.02, 0.0])
    near[0, 2], near[1, 2] = 1.3, -2.7
    rnd = np.eye(3) + rng.uniform(-0.05, 0.05, (3, 3)) * np.array([[1, 1, 0], [1, 1, 0], [0, 0, 0]])
    rnd[0, 2], rnd[1, 2] = rng.uniform(-5, 5), rng.uniform(-5, 5)
    rnd[2, :2] = rng.uniform(-2e-4, 2e-4, 2)
    flip = np.array([[-1.0, 0, w - 0.5], [0, -1.0, h - 0.5], [0, 0, 1.0]])
    cross = np.array([[1.0, 0, 0], [0, 1.0, 0], [0, -2.0 / h, 1.0]])       # z = 1 - 2y/h: 0 at mid-height
    return {"near": near, "random": rnd, "keystone": keystone(w, h, 0.45, 0.0, 0.05),
            "keystone_down": keystone(w, h, 0.0, 0.5, -0.1), "flip": flip, "negative_z": -rnd, "z_cross": cross}


def mosaic_with_holes(w, h, seed):
    """h×w×3 f32 in [0, 1) with Color::NO (-1) outside a ragged band, like an uncropped blend output."""
    rng = np.random.RandomState(seed)
    img = rng.rand(h, w, 3).astype(np.float32)
    yy, xx = np.mgrid[0:h, 0:w]
    top = h // 30 + (xx * 7 % 13)
    bottom = h - 1 - h // 40 - (xx * 5 % 11)
    img[(yy < top) | (yy > bottom)] = -1.0
    img[:, : max(1, w // 50)] = -1.0
    return img
