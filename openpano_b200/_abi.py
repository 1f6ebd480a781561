"""ctypes images of the structs in include/pano_b200.h."""
from __future__ import annotations

import ctypes as C


class PanoParams(C.Structure):
    _fields_ = [
        ("sift_working_size", C.c_int),
        ("num_octave", C.c_int),
        ("num_scale", C.c_int),
        ("scale_factor", C.c_float),
        ("gauss_sigma", C.c_float),
        ("gauss_window_factor", C.c_int),
        ("judge_extrema_diff_thres", C.c_float),
        ("contrast_thres", C.c_float),
        ("pre_color_thres", C.c_float),
        ("edge_ratio", C.c_float),
        ("calc_offset_depth", C.c_int),
        ("offset_thres", C.c_float),
        ("ori_radius", C.c_float),
        ("ori_hist_smooth_count", C.c_int),
        ("desc_hist_scale_factor", C.c_int),
        ("desc_int_factor", C.c_int),
        ("match_reject_next_ratio", C.c_float),
        ("focal_length", C.c_float),
        ("ordered_input", C.c_int),
        ("lazy_read", C.c_int),
        ("multiband", C.c_int),
        ("max_output_size", C.c_int),
    ]


def default_params(**overrides) -> PanoParams:
    """Defaults of the reference's config.cfg:2-69 (same values as
    pano_params_default in csrc/capi.cu)."""
    p = PanoParams(
        sift_working_size=800, num_octave=4, num_scale=7,
        scale_factor=1.4142135623, gauss_sigma=1.4142135623, gauss_window_factor=6,
        judge_extrema_diff_thres=2e-3, contrast_thres=4e-2, pre_color_thres=5e-2,
        edge_ratio=6.0, calc_offset_depth=4, offset_thres=0.5, ori_radius=4.5,
        ori_hist_smooth_count=2, desc_hist_scale_factor=3, desc_int_factor=512,
        match_reject_next_ratio=0.8, focal_length=37.0, ordered_input=0, lazy_read=1,
        multiband=0, max_output_size=8000,
    )
    for k, v in overrides.items():
        if not hasattr(p, k):
            raise AttributeError(f"pano_params has no field {k}")
        setattr(p, k, v)
    return p


class PanoSSPoint(C.Structure):
    _fields_ = [
        ("x", C.c_int), ("y", C.c_int),
        ("real_x", C.c_double), ("real_y", C.c_double),
        ("pyr_id", C.c_int), ("scale_id", C.c_int),
        ("dir", C.c_float), ("scale_factor", C.c_float),
    ]


class PanoBlendImage(C.Structure):
    _fields_ = [
        ("rgb_hwc", C.c_void_p),
        ("w", C.c_int), ("h", C.c_int),
        ("x0", C.c_int), ("y0", C.c_int), ("x1", C.c_int), ("y1", C.c_int),
        ("homo_inv", C.c_double * 9),
    ]


class PanoBlendGeom(C.Structure):
    _fields_ = [
        ("projection", C.c_int),
        ("res_x", C.c_double), ("res_y", C.c_double),
        ("proj_min_x", C.c_double), ("proj_min_y", C.c_double),
    ]


class PanoMatches(C.Structure):
    _fields_ = [
        ("n_pairs", C.c_int),
        ("count", C.POINTER(C.c_int)),
        ("offset", C.POINTER(C.c_int)),
        ("idx", C.POINTER(C.c_int)),
    ]


class PanoRansacPair(C.Structure):
    _fields_ = [
        ("n_match", C.c_int),
        ("kp1_xy", C.c_void_p), ("kp2_xy", C.c_void_p),
        ("n_hyp", C.c_int),
        ("homos", C.c_void_p),
        ("inlier_thres", C.c_float),
    ]


class PanoCylJob(C.Structure):
    _fields_ = [
        ("d_rgb_hwc", C.c_void_p), ("w", C.c_int), ("h", C.c_int),
        ("d_out_hwc", C.c_void_p), ("out_w", C.c_int), ("out_h", C.c_int),
        ("kpts_xy", C.c_void_p), ("n_kpts", C.c_int),
    ]


class PanoBaPair(C.Structure):
    _fields_ = [
        ("from_", C.c_int), ("to", C.c_int),
        ("match_begin", C.c_int), ("n_match", C.c_int),
        ("m", C.c_double * 9 * 13),
    ]


class PanoBaLink(C.Structure):
    _fields_ = [
        ("from_", C.c_int), ("to", C.c_int),
        ("match_begin", C.c_int), ("n_match", C.c_int),
    ]


PROJ_FLAT, PROJ_CYLINDRICAL, PROJ_SPHERICAL = 0, 1, 2
