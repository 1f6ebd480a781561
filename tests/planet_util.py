"""Checker wrappers and cases for the little-planet view, planet() (main.cc:294-331): orc_planet (the plain-C
restatement, oracle/liboracle_planet.so) and ref_planet (the reference's own planet(),
oracle/_ref/libopenpano_ref_planet.so), both built by oracle/planet.mk."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ORC_SO = ROOT / "oracle" / "liboracle_planet.so"
REF_SO = ROOT / "oracle" / "_ref" / "libopenpano_ref_planet.so"
SIZE = 1000                                  # main.cc:297 OUTSIZE
FIXTURE = "planet.npz"
_fp = C.POINTER(C.c_float)
_libs = {}

# name -> (w, h, seed, holes).  holes: "mosaic" = Color::NO outside a ragged band like an uncropped blend
# output; "band" = trailing NO columns, a NO row band and a strip whose green (not first) channel is negative;
# "" = none.  1449/1100 rows at 8000/6488 columns are the final mosaic sizes of the reference's two
# run_test.py targets; 1200 columns (a multiple of 4) put the j == 500 column on the exact integer columns
# w/4 and 3w/4; 2x2, 5x1 and 1x5 are the smallest inputs the reference takes (the last two give no colour).
CASES = {
    "mosaic_8000x1449": (8000, 1449, 31, "mosaic"),
    "mosaic_6488x1100": (6488, 1100, 32, "mosaic"),
    "holes_1800x300": (1800, 300, 33, "band"),
    "tall_600x800": (600, 800, 34, ""),
    "square_1000x1000": (1000, 1000, 35, "mosaic"),
    "w4_1200x400": (1200, 400, 36, ""),
    "tiny_2x2": (2, 2, 37, ""),
    "row_5x1": (5, 1, 38, ""),
    "column_1x5": (1, 5, 39, ""),
}
N_SAMPLE = 256


def _lib(path):
    if path not in _libs:
        if path == ORC_SO and not path.exists():
            subprocess.check_call(["make", "-s", "-C", str(ROOT / "oracle"), "-f", "planet.mk", "oracle"])
        _libs[path] = C.CDLL(str(path))
    return _libs[path]


def have_ref():
    return REF_SO.exists()


def make_input(w, h, seed, holes):
    """h×w×3 float32 in [0, 1) with Color::NO (-1) pixels as `holes` asks."""
    rng = np.random.RandomState(seed)
    img = rng.rand(h, w, 3).astype(np.float32)
    if holes == "mosaic":
        yy, xx = np.mgrid[0:h, 0:w]
        top = h // 40 + (xx * 7 % 113) * h // 1500
        bottom = h - 1 - h // 50 - (xx * 5 % 89) * h // 1200
        img[(yy < top) | (yy > bottom)] = -1.0
        img[:, : w // 200] = -1.0
    elif holes == "band":
        img[:, w - w // 18:] = -1.0
        img[h * 2 // 5: h * 2 // 5 + h // 15] = -1.0
        img[h // 6: h // 6 + 10, :, 1] = -1.0         # only channel 0 decides Color::NO
    return img


def case_input(name):
    return make_input(*CASES[name])


def sample_positions():
    """Fixed output pixels whose values the fixture stores whole, for locating a difference."""
    rng = np.random.RandomState(7)
    return rng.randint(0, SIZE, size=(N_SAMPLE, 2)).astype(np.int32)


def _run(fn, img):
    img = np.ascontiguousarray(img, np.float32)
    assert img.ndim == 3 and img.shape[2] == 3
    out = np.empty((SIZE, SIZE, 3), np.float32)
    fn.argtypes = [_fp, C.c_int, C.c_int, _fp]
    assert fn(img.ctypes.data_as(_fp), img.shape[1], img.shape[0], out.ctypes.data_as(_fp)) == 0
    return out


def orc_planet(img):
    """The restatement: planet()'s 1000×1000×3 float32 result for an H×W×3 float32 image."""
    return _run(_lib(ORC_SO).orc_planet, img)


def ref_planet(img):
    """The reference's own planet() on the same image."""
    return _run(_lib(REF_SO).ref_planet, img)
