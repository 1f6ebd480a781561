"""Blend geometries at the edges of the inverse map, and the f32 -> u8 value sweep.  Seeded, pure numpy.

A blend's inverse map (stitcher_image.cc:142-151) divides by rz, the depth of a canvas direction in the image's
camera frame.  Mild geometries keep rz near 1.  Here it reaches 0 and goes below it, and coordinates get infinite,
NaN or too big for an int:

* 360° rigs, cylindrical and spherical: N cameras yawed by 360°/N with alternating pitch, homo_inv = K·R
  (stitcher.cc:151).  Ranges, the canvas origin and the resolution are computed as update_proj_range and
  get_final_resolution do (stitcher_image.cc:40-111).  The image that straddles the ±π seam gets a range, and so
  an ROI, as wide as the canvas; its columns 90° off its axis are where rz crosses 0.
* A flat rig with wide yaw, whose outer images' corners lie behind the lens: their bounding boxes span rz = 0.
* Adversarial items added to a small translation stack, each with an ROI over the whole canvas: an all-zero
  homo_inv, rz = +0 along a canvas column, rz = -0.0, rz = 1e-300, constant coordinates at 2^31, 2147483520 (the
  largest float below it), in [2^31, 2^32) of both signs, on w-1 and h-1 and one double ulp below 0, NaN entries,
  a mirrored image, and a canvas with res_x != res_y.

Every case is (imgs, items, geom) in the form of synth.translation_blend_setup.
"""
from __future__ import annotations

import math

import numpy as np

from openpano_b200 import synth

CORNER_SAMPLE = 100      # stitcher_image.cc:42


def _corners():
    """update_proj_range's border samples in units of the image size (stitcher_image.cc:42-52)."""
    c = []
    for i in range(CORNER_SAMPLE):
        xi = i / CORNER_SAMPLE - 0.5
        c += [(xi, -0.5), (xi, 0.5)]
    for j in range(CORNER_SAMPLE):
        yj = j / CORNER_SAMPLE - 0.5
        c += [(-0.5, yj), (0.5, yj)]
    return np.array(c)


def homo2proj(projection, v):
    """projection.hh: (n, 3) homogeneous points -> (x, y) arrays."""
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    if projection == 0:
        return x / z, y / z
    if projection == 1:
        return np.arctan2(x, z), y / np.hypot(x, z)
    return np.arctan2(x, z), np.arctan2(y, np.hypot(x, z))


def blend_setup(homos, shapes, projection, identity=0, max_output_size=None, resolution=None):
    """items and geom of ConnectedImages::blend for cameras `homos` (image-centred pixel -> canvas direction) and
    image shapes (h, w).  resolution: (res_x, res_y) instead of get_final_resolution's."""
    corners = _corners()
    ranges = []
    for H, (h, w) in zip(homos, shapes):
        pts = np.stack([corners[:, 0] * w, corners[:, 1] * h, np.ones(len(corners))], 1) @ np.asarray(H).T
        px, py = homo2proj(projection, pts)
        ranges.append((px.min(), py.min(), px.max(), py.max()))
    pmin = (min(r[0] for r in ranges), min(r[1] for r in ranges))
    pmax = (max(r[2] for r in ranges), max(r[3] for r in ranges))
    if resolution is None:
        h, w = shapes[identity]
        H = np.asarray(homos[identity])
        c2 = homo2proj(projection, (H @ np.array([w / 2.0, h / 2.0, 1.0]))[None])
        c1 = homo2proj(projection, (H @ np.array([-w / 2.0, -h / 2.0, 1.0]))[None])
        rx, ry = float(c2[0][0] - c1[0][0]), float(c2[1][0] - c1[1][0])
        if projection != 0:
            rx = rx + 2 * math.pi if rx < 0 else rx
            ry = ry + math.pi if ry < 0 else ry
        res = [abs(rx) / w, abs(ry) / h]
        max_edge = max((pmax[0] - pmin[0]) / res[0], (pmax[1] - pmin[1]) / res[1])
        if max_output_size is not None and max_edge > max_output_size:
            ratio = float(np.float32(max_edge / max_output_size))     # `float ratio`, stitcher_image.cc:108
            res = [res[0] * ratio, res[1] * ratio]
    else:
        res = list(resolution)
    items = []
    for H, r in zip(homos, ranges):
        x0, y0 = int((r[0] - pmin[0]) / res[0]), int((r[1] - pmin[1]) / res[1])
        x1, y1 = int((r[2] - pmin[0]) / res[0]), int((r[3] - pmin[1]) / res[1])
        items.append((x0, y0, x1, y1, list(np.linalg.inv(np.asarray(H, np.float64)).ravel())))
    geom = dict(projection=projection, res_x=res[0], res_y=res[1], proj_min_x=pmin[0], proj_min_y=pmin[1])
    return items, geom


def _rot_y(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def _rot_x(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def _crops(n, w, h, seed):
    """n different w×h crops of one synth canvas."""
    canvas = synth.make_canvas(h + 40, w + 30 * n, seed)
    return [np.ascontiguousarray(canvas[(7 * k) % 40:(7 * k) % 40 + h, 30 * k:30 * k + w]) for k in range(n)]


def rig(projection, n=10, w=160, h=120, focal=150.0, pitch_deg=35.0, yaw0=0.1, seed=3, max_output_size=720):
    """A 360° rig (projection 1 or 2), or with projection 0 the wide flat rig: n cameras yawed from -70° to 70°."""
    imgs = _crops(n, w, h, seed)
    K = np.diag([focal, focal, 1.0])
    homos = []
    for k in range(n):
        if projection == 0:
            yaw, pitch = math.radians(-70.0 + 140.0 * k / (n - 1)), math.radians(4.0 * (k % 2) - 2.0)
        else:
            yaw, pitch = yaw0 + 2 * math.pi * k / n, math.radians(pitch_deg if k % 2 == 0 else -pitch_deg)
        R = _rot_x(pitch) @ _rot_y(-yaw)          # a canvas direction at (yaw, pitch) -> the camera axis
        homos.append(np.linalg.inv(K @ R))
    items, geom = blend_setup(homos, [im.shape[:2] for im in imgs], projection, identity=n // 2,
                              max_output_size=max_output_size)
    return imgs, items, geom


RIGS = {"cylindrical_360": (1,), "spherical_360": (2,), "flat_wide_yaw": (0,)}


# ----------------------------------------------------------------------------------------------- adversarial items
W, H = 160, 110


def _base():
    imgs, org = synth.make_stack(2, W, H, 70, 81)
    items, geom = synth.translation_blend_setup(org, W, H)
    return imgs, items, geom


def _whole_canvas(items):
    return 0, 0, max(it[2] for it in items), max(it[3] for it in items)


def _rows(ty=-20.0):
    """Second and third rows of an inverse map whose y varies over the canvas rows and whose rz is 1."""
    return [0.0, 1.0, ty, 0.0, 0.0, 1.0]


def _adv_homo(name, geom):
    """The homo_inv of adversarial item `name` on a flat canvas with `geom` (the image is W×H)."""
    col = geom["proj_min_x"] + 37 * geom["res_x"]                        # the canvas x of column 37
    hw = W * 0.5
    const_x = {
        "x_2p31": 2.0 ** 31, "x_2147483520": 2147483520.0, "x_2p31_plus": 2.0 ** 31 + 256, "x_3e9": 3e9,
        "x_2p32_minus": 2.0 ** 32 - 256, "x_neg_2p31": -2.0 ** 31, "x_neg_3e9": -3e9, "x_neg_2p32_minus": -(2.0 ** 32 - 256),
        "x_w_minus_1": W - 1.0, "x_below_w_minus_1": W - 1.0 - 2.0 ** -20, "x_ulp_below_0": None,
    }
    if name in const_x:
        x = const_x[name]
        t = np.nextafter(-hw, -np.inf) if x is None else x - hw    # x = t + w/2, exactly
        return [0.0, 0.0, float(t)] + _rows()
    if name.startswith("y_"):                             # the same constants for y, x varying
        x = {"y_2p31": 2.0 ** 31, "y_2147483520": 2147483520.0, "y_h_minus_1": H - 1.0, "y_neg_3e9": -3e9}[name]
        return [1.0, 0.0, -40.0, 0.0, 0.0, x - H * 0.5, 0.0, 0.0, 1.0]
    return {
        "nan_zero_homo": [0.0] * 9,                                       # rx = ry = rz = 0: NaN everywhere
        "nan_entry_x": [float("nan"), 0.0, -30.0] + _rows(),              # x NaN, y in range
        "nan_entry_z": [1.0, 0.0, -30.0, 0.0, 1.0, -20.0, 0.0, 0.0, float("nan")],
        "rz_zero_column": [1.0, 0.0, -col, 0.0, 1.0, 0.0, 1.0, 0.0, -col],   # rz = +0 (and rx = 0) at column 37
        "rz_zero_column_inf": [0.0, 0.0, 5.0, 0.0, 1.0, 0.0, 1.0, 0.0, -col],  # rz = +0, rx = 5: x = +inf there
        "rz_neg_zero": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, -0.0, -0.0, -0.0],  # rz = -0.0 where cx, cy > 0, else +0
        "rz_1e-300": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1e-300],    # |x| = inf but at cx = 0
        "mirrored": [-1.0, 0.0, 10.0, 0.0, 1.0, -15.0, 0.0, 0.0, 1.0],    # negative determinant
    }[name]


ADVERSARIAL = ["nan_zero_homo", "nan_entry_x", "nan_entry_z", "rz_zero_column", "rz_zero_column_inf", "rz_neg_zero",
               "rz_1e-300", "x_2p31", "x_2147483520", "x_2p31_plus", "x_3e9", "x_2p32_minus", "x_neg_2p31", "x_neg_3e9",
               "x_neg_2p32_minus", "x_w_minus_1", "x_below_w_minus_1", "x_ulp_below_0", "y_2p31", "y_2147483520",
               "y_h_minus_1", "y_neg_3e9", "mirrored", "res_xy"]


def adversarial(name):
    """The base stack plus one adversarial image (a third crop) whose ROI is the whole canvas; "res_xy" is the base
    stack alone on a canvas with res_x = 1 and res_y = 1.5."""
    imgs, items, geom = _base()
    if name == "res_xy":
        org = [(0.0, 0.0), (70.0, 0.0)]
        homos = [np.array([[1.0, 0, x], [0, 1.0, y], [0, 0, 1.0]]) for x, y in org]
        items, geom = blend_setup(homos, [(H, W)] * 2, 0, resolution=(1.0, 1.5))
        return imgs, items, geom
    extra = synth.make_canvas(H, W, 82)
    items = items + [_whole_canvas(items) + (_adv_homo(name, geom),)]
    return imgs + [extra], items, geom


def geometry(name):
    if name in RIGS:
        return rig(*RIGS[name])
    return adversarial(name)


GEOMETRIES = list(RIGS) + ADVERSARIAL


def only_nan(name):
    """True for the cases whose coordinates are finite and in int range or NaN, never ±inf or >= 2^31."""
    return name.startswith("nan_")


# ----------------------------------------------------------------------------------------------- f32 -> u8 sweep
def u8_sweep_values():
    """Mosaic samples at the edges of write_rgb's (v < 0 ? 1 : v) * 255 truncation: every k/255 and its float
    neighbours, every float in [1, 256/255], 2^31/255 and 2^32/255 with their neighbours, ±inf, NaN, -0.0,
    denormals, negatives and large values."""
    f = np.float32
    vals = []
    for k in range(257):
        v = f(k) / f(255)
        vals += [np.nextafter(v, f(-np.inf)), v, np.nextafter(v, f(np.inf))]
        vals.append(f(k / 255.0))
    lo, hi = f(1.0).view(np.int32), (f(256) / f(255)).view(np.int32)
    vals += list(np.arange(lo, hi + 2, dtype=np.int32).view(np.float32))
    for big in (2.0 ** 31 / 255, 2.0 ** 32 / 255, 2.0 ** 24 / 255, 2.0 ** 31, 1e10):
        v = f(big)
        for _ in range(4):
            v = np.nextafter(v, f(-np.inf))
        for _ in range(9):
            vals.append(v)
            v = np.nextafter(v, f(np.inf))
    vals += [f(np.inf), f(-np.inf), f(np.nan), f(-np.nan), f(-0.0), f(0.0), np.finfo(np.float32).max,
             -np.finfo(np.float32).max, f(1e-45), f(-1e-45), np.finfo(np.float32).tiny, f(-1e-40), f(-1.0), f(-0.5),
             f(-1e-30), f(-2.0 ** 31), f(1e-40), f(255.0), f(256.0), f(2.0 ** 24)]
    return np.array(vals, np.float32)


def u8_sweep_mosaic(w=97):
    """The sweep values as an h×w×3 float32 mosaic, each value in every channel position; zero padding."""
    v = u8_sweep_values()
    v = np.concatenate([v, np.roll(v, 1), np.roll(v, 2)])
    n = -(-len(v) // (w * 3)) * w * 3
    out = np.zeros(n, np.float32)
    out[:len(v)] = v
    return out.reshape(-1, w, 3)


def x86_write_rgb(mat):
    """write_rgb's conversion as x86-64 computes it: the float product (v < 0 ? 1 : v) * 255, cvttss2si (INT_MIN
    for NaN and outside [-2^31, 2^31)), the low byte."""
    with np.errstate(over="ignore", invalid="ignore"):
        v = np.where(mat < 0, np.float32(1), mat).astype(np.float32) * np.float32(255)
    ok = (v >= -2.0 ** 31) & (v < 2.0 ** 31)
    i = np.where(ok, np.trunc(np.where(ok, v, 0)).astype(np.int64), -2 ** 31)
    return (i & 0xFF).astype(np.uint8)
