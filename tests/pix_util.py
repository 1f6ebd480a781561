"""Checker wrappers and cases for the reference's decoder and encoder layouts (lib/imgio.cc): the plain-C
restatement (oracle/liboracle_pix.so: orc_read_png_rgba, orc_read_img_planar, orc_write_png_rgba,
orc_write_rgb_planar) and the reference's read_img / write_rgb with its own lodepng and CImg
(oracle/_ref/libopenpano_ref_pix.so), both built by oracle/pix_formats.mk."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ORC_SO = ROOT / "oracle" / "liboracle_pix.so"
REF_SO = ROOT / "oracle" / "_ref" / "libopenpano_ref_pix.so"
_fp = C.POINTER(C.c_float)
_up = C.POINTER(C.c_ubyte)
_libs = {}

# lodepng colour types (LodePNGColorType) and the bit depths written for each PNG case
LCT_GREY, LCT_RGB, LCT_PALETTE, LCT_GREY_ALPHA, LCT_RGBA = 0, 2, 3, 4, 6
# name -> (colour type, bit depth): every colour type read_png meets, 8-bit, plus 16-bit RGB and grey
PNG_CASES = {
    "grey": (LCT_GREY, 8),
    "grey_alpha": (LCT_GREY_ALPHA, 8),
    "rgb": (LCT_RGB, 8),
    "rgba": (LCT_RGBA, 8),
    "palette": (LCT_PALETTE, 8),
    "rgb16": (LCT_RGB, 16),
    "grey16": (LCT_GREY, 16),
}
_SAMPLES = {LCT_GREY: 1, LCT_RGB: 3, LCT_PALETTE: 1, LCT_GREY_ALPHA: 2, LCT_RGBA: 4}


def _lib(path):
    if path not in _libs:
        if path == ORC_SO and not path.exists():
            subprocess.check_call(["make", "-s", "-C", str(ROOT / "oracle"), "-f", "pix_formats.mk", "oracle"])
        _libs[path] = C.CDLL(str(path))
    return _libs[path]


def have_ref():
    return REF_SO.exists()


def png_raw(name, w, h, seed):
    """(raw bytes, colour type, bit depth, palette or None) of a w×h PNG case: random samples (16-bit ones
    big-endian, as PNG stores them), palette indices into a random 256-entry RGBA palette."""
    ct, bd = PNG_CASES[name]
    rng = np.random.RandomState(seed)
    raw = rng.randint(0, 256, size=h * w * _SAMPLES[ct] * (bd // 8)).astype(np.uint8)
    pal = rng.randint(0, 256, size=(256, 4)).astype(np.uint8) if ct == LCT_PALETTE else None
    return raw, ct, bd, pal


def ref_read_png(name, w, h, seed):
    """The reference's file path for PNG case `name`: (read_img's h×w×3 float32, lodepng::decode's h×w×4 uint8)."""
    raw, ct, bd, pal = png_raw(name, w, h, seed)
    out = np.empty((h, w, 3), np.float32)
    rgba = np.empty((h, w, 4), np.uint8)
    fn = _lib(REF_SO).ref_read_png
    fn.argtypes = [_up, C.c_int, C.c_int, C.c_int, C.c_int, _up, C.c_int, _fp, _up]
    pal_p = pal.ctypes.data_as(_up) if pal is not None else None
    rc = fn(raw.ctypes.data_as(_up), w, h, ct, bd, pal_p, 0 if pal is None else len(pal), out.ctypes.data_as(_fp),
            rgba.ctypes.data_as(_up))
    assert rc == 0, f"ref_read_png({name}) failed"
    return out, rgba


def ref_read_cimg(pix):
    """read_img and CImg<unsigned char> on a PPM (H×W×3) or PGM (H×W) file of pix: (h×w×3 float32, planes
    (3, h, w) or (h, w))."""
    pix = np.ascontiguousarray(pix, np.uint8)
    h, w = pix.shape[:2]
    ch = 1 if pix.ndim == 2 else 3
    out = np.empty((h, w, 3), np.float32)
    planes = np.empty((ch, h, w) if ch == 3 else (h, w), np.uint8)
    fn = _lib(REF_SO).ref_read_cimg
    fn.argtypes = [_up, C.c_int, C.c_int, C.c_int, _fp, _up]
    assert fn(pix.ctypes.data_as(_up), w, h, ch, out.ctypes.data_as(_fp), planes.ctypes.data_as(_up)) == 0
    return out, planes


def _write(lib, name, mat, shape):
    mat = np.ascontiguousarray(mat, np.float32)
    h, w = mat.shape[:2]
    out = np.empty(shape(h, w), np.uint8)
    fn = getattr(_lib(lib), name)
    fn.argtypes = [_fp, C.c_int, C.c_int, _up]
    assert fn(mat.ctypes.data_as(_fp), w, h, out.ctypes.data_as(_up)) == 0, name
    return out


def ref_write_png(mat):
    """write_rgb(".png") of an H×W×3 float32 mosaic, decoded back by lodepng: (h, w, 4) uint8."""
    return _write(REF_SO, "ref_write_png", mat, lambda h, w: (h, w, 4))


def ref_write_cimg(mat):
    """write_rgb(".ppm") of the mosaic, loaded back by CImg: its planes, (3, h, w) uint8."""
    return _write(REF_SO, "ref_write_cimg", mat, lambda h, w: (3, h, w))


def orc_write_png_rgba(mat):
    return _write(ORC_SO, "orc_write_png_rgba", mat, lambda h, w: (h, w, 4))


def orc_write_rgb_planar(mat):
    return _write(ORC_SO, "orc_write_rgb_planar", mat, lambda h, w: (3, h, w))


def _read(name, pix, h, w):
    pix = np.ascontiguousarray(pix, np.uint8)
    out = np.empty((h, w, 3), np.float32)
    fn = getattr(_lib(ORC_SO), name)
    fn.argtypes = [_up, C.c_int, C.c_int, _fp]
    assert fn(pix.ctypes.data_as(_up), w, h, out.ctypes.data_as(_fp)) == 0, name
    return out


def orc_read_png_rgba(rgba):
    """read_png on lodepng's (h, w, 4) buffer: h×w×3 float32."""
    return _read("orc_read_png_rgba", rgba, rgba.shape[0], rgba.shape[1])


def orc_read_img_planar(planes):
    """read_img's spectrum-3 path on CImg's (3, h, w) planes: h×w×3 float32."""
    return _read("orc_read_img_planar", planes, planes.shape[1], planes.shape[2])


def to_rgba(rgb, alpha_seed=None):
    """Interleaved h×w×3 pixels in lodepng's layout; the fourth byte random (alpha_seed) or 255."""
    h, w = rgb.shape[:2]
    out = np.empty((h, w, 4), np.uint8)
    out[..., :3] = rgb
    out[..., 3] = 255 if alpha_seed is None else np.random.RandomState(alpha_seed).randint(0, 256, size=(h, w))
    return out


def to_planar(rgb):
    """Interleaved h×w×3 pixels in CImg's layout: (3, h, w)."""
    return np.ascontiguousarray(np.moveaxis(rgb, 2, 0))


def mosaic_with_holes(h, w, seed):
    """An h×w×3 float32 mosaic with Color::NO (-1) pixels, as a blend leaves them."""
    rng = np.random.RandomState(seed)
    m = rng.rand(h, w, 3).astype(np.float32)
    m[: h // 7] = -1.0
    m[:, w - w // 9:] = -1.0
    m[h // 2, w // 3: w // 2, 1] = -1.0
    return m
