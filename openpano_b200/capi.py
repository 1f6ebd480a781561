"""ctypes binding of libpano_b200.so (include/pano_b200.h).

There is no CPU fallback: if the CUDA library is missing this module raises at
import, and if no H100 is visible `Engine()` raises PanoError (PANO_ERR_NO_DEVICE).
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

from ._abi import (PanoBaLink, PanoBaPair, PanoBlendGeom, PanoCylJob, PanoBlendImage, PanoMatches, PanoParams, PanoRansacPair, PanoSSPoint,
                   default_params)

LIB_PATH = Path(__file__).resolve().parent / "libpano_b200.so"

_fp = C.POINTER(C.c_float)
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_vpp = C.POINTER(C.c_void_p)

SSPOINT_DTYPE = np.dtype([("x", "<i4"), ("y", "<i4"), ("real_x", "<f8"), ("real_y", "<f8"),
                          ("pyr_id", "<i4"), ("scale_id", "<i4"), ("dir", "<f4"),
                          ("scale_factor", "<f4")], align=True)


class PanoError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"pano_b200 error {code}: {msg}")
        self.code = code


def _load():
    if not LIB_PATH.exists():
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). openpano_b200 has no CPU fallback.")
    # PANO_B200_LIB: development override to A/B a differently tuned build of the same library
    lib = C.CDLL(os.environ.get("PANO_B200_LIB", str(LIB_PATH)), mode=os.RTLD_LOCAL)
    P = C.POINTER(PanoParams)
    sig = {
        "pano_params_default": (None, [P]),
        "pano_create": (C.c_int, [_vpp, C.c_int, C.c_void_p]),
        "pano_destroy": (None, [C.c_void_p]),
        "pano_last_error": (C.c_char_p, [C.c_void_p]),
        "pano_sync": (C.c_int, [C.c_void_p]),
        "pano_stream": (C.c_void_p, [C.c_void_p]),
        "pano_profile_enable": (C.c_int, [C.c_void_p, C.c_int]),
        "pano_profile_reset": (C.c_int, [C.c_void_p]),
        "pano_profile_read": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p, _ip, _dp]),
        "pano_launch_count": (C.c_longlong, [C.c_void_p]),
        "pano_trim": (C.c_int, [C.c_void_p]),
        "pano_match_last_exact_rows": (C.c_int, [C.c_void_p]),
        "pano_match_last_nominated_rows": (C.c_int, [C.c_void_p]),
        "pano_sift_detect_batch": (C.c_int, [C.c_void_p, C.c_int, _vpp, _ip, _ip, P, _vpp]),
        "pano_sift_detect_batch_dev": (C.c_int, [C.c_void_p, C.c_int, _vpp, _ip, _ip, P, _vpp]),
        "pano_sift_detect": (C.c_int, [C.c_void_p, _fp, C.c_int, C.c_int, P, _vpp]),
        "pano_sift_detect_batch_rgb8": (C.c_int, [C.c_void_p, C.c_int, _vpp, _ip, _ip, _ip, P, _vpp]),
        "pano_sift_detect_batch_rgb8_dev": (C.c_int, [C.c_void_p, C.c_int, _vpp, _ip, _ip, _ip, P, _vpp]),
        "pano_featureset_upload": (C.c_int, [C.c_void_p, C.c_int, _ip, _vpp, _vpp, _vpp]),
        "pano_featureset_num_images": (C.c_int, [C.c_void_p]),
        "pano_featureset_count": (C.c_int, [C.c_void_p, C.c_int]),
        "pano_featureset_download": (C.c_int, [C.c_void_p, C.c_int, _dp, _fp]),
        "pano_featureset_download_real": (C.c_int, [C.c_void_p, C.c_int, _dp]),
        "pano_featureset_free": (None, [C.c_void_p]),
        "pano_match_pairs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, _ip, P, C.POINTER(PanoMatches)]),
        "pano_matches_free": (None, [C.POINTER(PanoMatches)]),
        "pano_match_pairs_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, _ip, P, _ip]),
        "pano_match_pairs_shard": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, _ip, P, C.c_int, C.c_int, C.POINTER(PanoMatches)]),
        "pano_match_pairs_dev_shard": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, _ip, P, C.c_int, C.c_int, _ip]),
        "pano_match_bruteforce": (C.c_int, [C.c_void_p, _fp, C.c_int, _fp, C.c_int, P, _ip, _ip]),
        "pano_comm_unique_id": (C.c_int, [C.c_char_p]),
        "pano_comm_create": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_char_p, _vpp]),
        "pano_comm_adopt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, _vpp]),
        "pano_comm_destroy": (None, [C.c_void_p]),
        "pano_comm_world": (C.c_int, [C.c_void_p]),
        "pano_comm_rank": (C.c_int, [C.c_void_p]),
        "pano_comm_allgather_features": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, _vpp]),
        "pano_comm_allgather_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
        "pano_ransac_score_pairs": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoRansacPair), _ip, _ip, _vpp, _vpp]),
        "pano_ba_jacobian": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(PanoBaPair), _dp, _dp, _dp]),
        "pano_ba_session_create": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(PanoBaLink), _dp, _vpp]),
        "pano_ba_session_free": (None, [C.c_void_p]),
        "pano_ba_error": (C.c_int, [C.c_void_p, C.c_int, _dp, _dp, _dp, _dp]),
        "pano_ba_normal_equations": (C.c_int, [C.c_void_p, C.c_int, _dp, _dp, _dp, _dp]),
        "pano_cyl_warp_shape": (C.c_int, [C.c_int, C.c_int, C.c_double, P, _ip, _ip, _dp, _dp]),
        "pano_cyl_warp": (C.c_int, [C.c_void_p, _fp, C.c_int, C.c_int, C.c_double, P, _fp, C.c_int,
                                    C.c_int, _dp, C.c_int]),
        "pano_cyl_warp_batch_dev": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoCylJob), C.c_double, P]),
        "pano_cyl_warp_batch_rgb8_dev": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoCylJob), _vpp, _ip, C.c_double,
                                                   P]),
        "pano_blend_target_size": (C.c_int, [C.c_int, C.POINTER(PanoBlendImage), _ip, _ip]),
        "pano_blend": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage), C.POINTER(PanoBlendGeom),
                                 C.c_int, P, _fp, C.c_int, C.c_int]),
        "pano_blend_dev": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage),
                                     C.POINTER(PanoBlendGeom), C.c_int, P, C.c_void_p, C.c_int, C.c_int]),
        "pano_blend_rgb8_dev": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage), _vpp, _ip,
                                          C.POINTER(PanoBlendGeom), C.c_int, P, C.c_void_p, C.c_int, C.c_int]),
        "pano_blend_rows_dev": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage), C.POINTER(PanoBlendGeom),
                                          C.c_int, P, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
        "pano_blend_rows_rgb8_dev": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage), _vpp, _ip,
                                               C.POINTER(PanoBlendGeom), C.c_int, P, C.c_void_p, C.c_int, C.c_int,
                                               C.c_int, C.c_int]),
        "pano_blend_stream_create": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage), C.POINTER(PanoBlendGeom),
                                               C.c_int, P, C.c_int, C.c_int, _vpp]),
        "pano_blend_stream_add": (C.c_int, [C.c_void_p, C.c_int, C.c_int, _vpp, C.c_int, C.c_int]),
        "pano_blend_stream_finish_dev": (C.c_int, [C.c_void_p, C.c_void_p]),
        "pano_blend_stream_finish": (C.c_int, [C.c_void_p, _fp]),
        "pano_blend_stream_free": (None, [C.c_void_p]),
        "pano_blend_stream_create_rows": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage),
                                                    C.POINTER(PanoBlendGeom), C.c_int, P, C.c_int, C.c_int, C.c_int,
                                                    C.c_int, _vpp]),
        "pano_blend_stream_needs": (C.c_int, [C.c_void_p, C.c_void_p]),
        "pano_blend_stream_create_cyl": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage), _ip, _ip, C.c_double,
                                                   C.POINTER(PanoBlendGeom), C.c_int, P, C.c_int, C.c_int, _vpp]),
        "pano_blend_sweep_plan": (C.c_int, [C.c_int, C.POINTER(PanoBlendImage), C.POINTER(PanoBlendGeom), C.c_int, P,
                                            C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t), C.c_size_t, _ip,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_longlong),
                                            C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]),
        "pano_blend_sweep_create": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage), C.POINTER(PanoBlendGeom),
                                              C.c_int, P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t),
                                              C.c_size_t, C.c_int, _vpp]),
        "pano_blend_sweep_next": (C.c_int, [C.c_void_p, C.c_void_p]),
        "pano_blend_sweep_strip": (C.c_int, [C.c_void_p, _vpp, _ip, C.c_int]),
        "pano_blend_sweep_finish_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, _ip]),
        "pano_blend_sweep_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_ulonglong),
                                             C.POINTER(C.c_ulonglong)]),
        "pano_blend_sweep_free": (None, [C.c_void_p]),
        "pano_blend_sweep_plan_cyl": (C.c_int, [C.c_int, C.POINTER(PanoBlendImage), C.POINTER(PanoBlendGeom), C.c_int,
                                                P, C.c_int, C.c_int, _dp, C.c_int, C.POINTER(C.c_size_t), C.c_size_t,
                                                _ip, _ip, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.POINTER(C.c_longlong), C.POINTER(C.c_ulonglong),
                                                C.POINTER(C.c_ulonglong)]),
        "pano_blend_sweep_create_cyl": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PanoBlendImage), _ip, _ip,
                                                  C.c_double, C.POINTER(PanoBlendGeom), C.c_int, P, C.c_int, C.c_int,
                                                  _dp, C.c_int, C.POINTER(C.c_size_t), C.c_size_t, C.c_int, _vpp]),
        "pano_sift_stream_create": (C.c_int, [C.c_void_p, C.c_int, _ip, _ip, P, _vpp]),
        "pano_sift_stream_add": (C.c_int, [C.c_void_p, C.c_int, C.c_int, _vpp, C.c_int, C.c_int]),
        "pano_sift_stream_finish": (C.c_int, [C.c_void_p, _vpp]),
        "pano_sift_stream_free": (None, [C.c_void_p]),
        "pano_mem_high_water": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t), C.c_int]),
        "pano_planet": (C.c_int, [C.c_void_p, _fp, C.c_int, C.c_int, _fp]),
        "pano_planet_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
        "pano_planet_pix8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, _fp]),
        "pano_planet_pix8_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
        "pano_featureset_import_dev": (C.c_int, [C.c_void_p, C.c_int, _ip, _vpp, _vpp, _vpp]),
        "pano_featureset_export_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
        "pano_featureset_export_all_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
        "pano_rgb8_to_mat32f_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
        "pano_rgb8_to_mat32f_batch_dev": (C.c_int, [C.c_void_p, C.c_int, _vpp, _ip, _ip, _ip, _vpp]),
        "pano_crop_rect_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
        "pano_crop_scan_create": (C.c_int, [C.c_void_p, C.c_int, C.c_int, _vpp]),
        "pano_crop_scan_add_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
        "pano_crop_scan_rect": (C.c_int, [C.c_void_p, _ip]),
        "pano_crop_scan_free": (None, [C.c_void_p]),
        "pano_rgb8_crop_to_pix8_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                                 C.c_void_p]),
        "pano_mat32f_to_rgb8_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
        "pano_mat32f_to_pix8_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                              C.c_void_p]),
        "pano_dev_alloc": (C.c_int, [C.c_void_p, C.c_size_t, _vpp]),
        "pano_dev_free": (C.c_int, [C.c_void_p, C.c_void_p]),
        "pano_dev_upload": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
        "pano_dev_download": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
        "pano_dev_upload_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
        "pano_dev_download_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
        "pano_host_alloc": (C.c_int, [C.c_size_t, _vpp]),
        "pano_host_free": (C.c_int, [C.c_void_p]),
        "pano_event_create": (C.c_int, [C.c_void_p, _vpp]),
        "pano_event_record": (C.c_int, [C.c_void_p, C.c_void_p]),
        "pano_event_wait": (C.c_int, [C.c_void_p, C.c_void_p]),
        "pano_event_sync": (C.c_int, [C.c_void_p]),
        "pano_event_destroy": (None, [C.c_void_p]),
        "pano_sift_trace_run": (C.c_int, [C.c_void_p, _fp, C.c_int, C.c_int, P, _vpp]),
        "pano_sift_trace_working_size": (C.c_int, [C.c_void_p, _ip, _ip]),
        "pano_sift_trace_octave_size": (C.c_int, [C.c_void_p, C.c_int, _ip, _ip]),
        "pano_sift_trace_plane": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, _fp]),
        "pano_sift_trace_points": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(PanoSSPoint)]),
        "pano_sift_trace_descriptors": (C.c_int, [C.c_void_p, C.c_int, _dp, _fp]),
        "pano_sift_trace_free": (None, [C.c_void_p]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)  # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    return lib, sorted(sig)


LIB, EXPORTED = _load()


def _f(a):
    return a.ctypes.data_as(_fp)


def _d(a):
    return a.ctypes.data_as(_dp)


def _i(a):
    return a.ctypes.data_as(_ip)


class _Handle:
    """Owns one engine handle (self._h, freed by _FREE): close() frees it once, and so does garbage collection, which
    swallows errors.  _call raises the context's error for a non-zero return code."""
    _FREE = None

    def _call(self, rc):
        self.eng._check(rc)

    def close(self):
        if self._h:
            type(self)._FREE(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class FeatureSet(_Handle):
    """Device-resident descriptors + coordinates of a batch of images."""
    _FREE = LIB.pano_featureset_free

    def __init__(self, eng, handle):
        self.eng, self._h = eng, handle

    @property
    def n_images(self):
        return LIB.pano_featureset_num_images(self._h)

    def count(self, i):
        n = LIB.pano_featureset_count(self._h, i)
        if n < 0:
            self.eng._raise(n)
        return n

    def download(self, i):
        n = self.count(i)
        coor = np.zeros((n, 2), np.float64)
        desc = np.zeros((n, 128), np.float32)
        self.eng._check(LIB.pano_featureset_download(self._h, i, _d(coor), _f(desc)))
        return coor, desc

    def export_all_dev(self, d_coor, d_desc):
        """Every image's rows packed back to back into device buffers (one launch)."""
        self.eng._check(LIB.pano_featureset_export_all_dev(self._h, C.c_void_p(d_coor or 0), C.c_void_p(d_desc or 0)))

    def export_dev(self, i, d_coor, d_desc):
        """Device-to-device copy of image i's rows (coordinates n×2 f64, descriptors n×128 f32)."""
        self.eng._check(LIB.pano_featureset_export_dev(self._h, i, C.c_void_p(d_coor or 0), C.c_void_p(d_desc or 0)))

    free = _Handle.close


class GpuSiftTrace(_Handle):
    _FREE = LIB.pano_sift_trace_free

    def __init__(self, eng, handle):
        self.eng, self._h = eng, handle

    def working_size(self):
        w, h = C.c_int(), C.c_int()
        LIB.pano_sift_trace_working_size(self._h, C.byref(w), C.byref(h))
        return w.value, h.value

    def octave_size(self, o):
        w, h = C.c_int(), C.c_int()
        self.eng._check(LIB.pano_sift_trace_octave_size(self._h, o, C.byref(w), C.byref(h)))
        return w.value, h.value

    def plane(self, kind, octave=0, level=0):
        if kind == 0:
            w, h = self.working_size()
            out = np.empty((h, w, 3), np.float32)
        else:
            w, h = self.octave_size(octave)
            out = np.empty((h, w), np.float32)
        self.eng._check(LIB.pano_sift_trace_plane(self._h, kind, octave, level, _f(out)))
        return out

    def points(self, stage):
        n = LIB.pano_sift_trace_points(self._h, stage, 0, None)
        if n < 0:
            self.eng._raise(n)
        out = np.zeros(n, SSPOINT_DTYPE)
        if n:
            LIB.pano_sift_trace_points(self._h, stage, n, out.ctypes.data_as(C.POINTER(PanoSSPoint)))
        return out

    def descriptors(self):
        n = LIB.pano_sift_trace_descriptors(self._h, 0, None, None)
        if n < 0:
            self.eng._raise(n)
        coor = np.zeros((n, 2), np.float64)
        desc = np.zeros((n, 128), np.float32)
        if n:
            LIB.pano_sift_trace_descriptors(self._h, n, _d(coor), _f(desc))
        return coor, desc


class BaSession(_Handle):
    """Device-resident state of one bundle adjustment (pano_ba_session): the match coordinates, J and the
    residuals of the last error() call.  error() is calcError + update_stats; normal_equations() is
    get_param_update up to the damping, with b = J^T times the residuals of the LAST error() call."""
    _FREE = LIB.pano_ba_session_free

    def __init__(self, eng, handle, n_cam, n_pair, n_match):
        self.eng, self._h = eng, handle
        self.n_cam, self.n_pair, self.n_match = n_cam, n_pair, n_match

    def _mats(self, a, per_pair, what):
        a = np.ascontiguousarray(a, np.float64)
        if a.size != self.n_pair * per_pair:
            raise PanoError(-2, f"ba session: {what} has {a.size} doubles, the session's {self.n_pair} pairs need "
                                f"{self.n_pair * per_pair}")
        return a.reshape(-1)

    def error(self, hto, want_residuals=True):
        """hto: [n_pair, 9] Hto_to_from of the state.  -> (avg, max, residuals [2 n_match] or None)."""
        h = self._mats(hto, 9, "hto")
        avg, mx = C.c_double(), C.c_double()
        res = np.zeros(max(2 * self.n_match, 1), np.float64) if want_residuals else None
        self.eng._check(LIB.pano_ba_error(self._h, self.n_pair, _d(h) if h.size else None, C.byref(avg), C.byref(mx),
                                          _d(res) if want_residuals else None))
        return avg.value, mx.value, (res[:2 * self.n_match] if want_residuals else None)

    def normal_equations(self, mats, want_rows=False):
        """mats: [n_pair, 13, 9] in pano_ba_pair.m order.  -> (jtj [6n, 6n] undamped, b [6n], j_rows [n_match, 24] or None)."""
        m = self._mats(mats, 117, "mats")
        n = 6 * self.n_cam
        jtj = np.full((n, n), np.nan, np.float64)
        b = np.full(n, np.nan, np.float64)
        rows = np.zeros((max(self.n_match, 1), 24), np.float64) if want_rows else None
        self.eng._check(LIB.pano_ba_normal_equations(self._h, self.n_pair, _d(m) if m.size else None, _d(jtj), _d(b),
                                                     _d(rows) if want_rows else None))
        return jtj, b, (rows[:self.n_match] if want_rows else None)


# pano_src_kind
SRC_F32_DEV, SRC_F32_HOST, SRC_RGB8_DEV, SRC_RGB8_HOST = 0, 1, 2, 3

# PANO_PIX_*: the pixel formats of decoded 8-bit images, passed where the 8-bit entry points take `channels`
PIX_GREY, PIX_RGB, PIX_RGBA, PIX_RGB_PLANAR = 1, 3, 0x104, 0x203
# the `fmt` keyword of the numpy methods: "rgba" selects lodepng's H×W×4 buffers, "planar" CImg's 3×H×W planes;
# None keeps the inference from the shape (H×W or H×W×1 grey, H×W×3 interleaved RGB)
PIX_FORMATS = {"grey": PIX_GREY, "rgb": PIX_RGB, "rgba": PIX_RGBA, "planar": PIX_RGB_PLANAR}


def pix_format(a, fmt=None):
    """(PANO_PIX_* code, h, w) of a uint8 array read in layout `fmt`; raises PanoError if the shape does not fit."""
    if fmt is None:
        if a.ndim == 2 or (a.ndim == 3 and a.shape[2] == 1):
            return PIX_GREY, a.shape[0], a.shape[1]
        if a.ndim == 3 and a.shape[2] == 3:
            return PIX_RGB, a.shape[0], a.shape[1]
    elif fmt not in PIX_FORMATS:
        raise PanoError(-2, f"unknown pixel format {fmt!r} (one of {sorted(PIX_FORMATS)})")
    elif fmt == "planar":
        if a.ndim == 3 and a.shape[0] == 3:
            return PIX_RGB_PLANAR, a.shape[1], a.shape[2]
    else:
        code = PIX_FORMATS[fmt]
        if code == PIX_GREY and a.ndim == 2:
            return code, a.shape[0], a.shape[1]
        if a.ndim == 3 and a.shape[2] == {PIX_GREY: 1, PIX_RGB: 3, PIX_RGBA: 4}[code]:
            return code, a.shape[0], a.shape[1]
    raise PanoError(-2, f"8-bit source of shape {a.shape} does not fit format {fmt or 'grey / rgb'}: expected H×W or "
                        "H×W×{1,3}, H×W×4 with fmt='rgba', 3×H×W with fmt='planar'")


def _fmt_list(fmt, n):
    return list(fmt) if isinstance(fmt, (list, tuple)) else [fmt] * n


class _SourceStream(_Handle):
    """What the windowed streams share: add() takes numpy arrays (host; uint8 H×W / H×W×1 / H×W×3 or float32
    H×W×3, the kind from the dtype) or raw pointers with an explicit kind (SRC_*).  Every failure is sticky, as
    in the C ABI."""
    _NAME = ""
    _ADD = None
    _NULL_OK = False     # None in a numpy window: an image the stream does not read (row-strip blend streams)

    def __init__(self, eng, handle, shapes):
        self.eng, self._h = eng, handle
        self.shapes = list(shapes)
        self.added = 0
        self._err = None

    def _fail(self, msg):
        self._err = PanoError(-2, msg)
        raise self._err

    def _call(self, rc):
        if rc != 0:
            self._err = PanoError(rc, LIB.pano_last_error(self.eng._h).decode())
            raise self._err

    def add(self, srcs, kind=None, channels=None, fmt=None):
        """Adds the next len(srcs) images.  fmt ("rgba" or "planar", see pix_format) reads uint8 arrays in that
        layout; raw pointers take a PANO_PIX_* code as `channels`."""
        if self._err is not None:
            raise self._err
        keep = []
        if kind is None:
            all_srcs = list(srcs)
            arrs = [a for a in all_srcs if a is not None] if self._NULL_OK else all_srcs
            dts = {a.dtype for a in arrs}
            if len(dts) > 1 or (not dts and not all_srcs) or (dts and dts.pop() not in (np.uint8, np.float32)):
                self._fail(f"{self._NAME}: sources must all be uint8 or all float32 numpy arrays")
            u8 = bool(arrs) and arrs[0].dtype == np.uint8
            kind = SRC_RGB8_HOST if u8 else SRC_F32_HOST
            channels = None
            for k, a in enumerate(all_srcs):
                if a is None:
                    keep.append(None)
                    continue
                want = self.shapes[self.added + k] if self.added + k < len(self.shapes) else None
                if u8 and fmt is not None:
                    try:
                        ch, ah, aw = pix_format(a, fmt)
                    except PanoError as e:
                        self._fail(f"{self._NAME}: source {self.added + k}: {e}")
                    a_hw = (ah, aw)
                else:
                    ch = 1 if a.ndim == 2 else (a.shape[2] if a.ndim == 3 else -1)
                    a_hw = a.shape[:2]
                if want is None or a_hw != tuple(want) or (ch not in (1, 3) if u8 and fmt is None else
                                                           (not u8 and ch != 3)) or \
                        (channels is not None and ch != channels):
                    self._fail(f"{self._NAME}: source {self.added + k} has shape {a.shape}, the stream expects "
                               f"{want} with {'1 or 3 channels' if u8 else '3 channels'}, the same for the window")
                channels = ch
                keep.append(np.ascontiguousarray(a))
            ptrs = [a.ctypes.data if a is not None else 0 for a in keep]
            channels = 3 if channels is None else channels
        else:
            ptrs = [int(p or 0) for p in srcs]
            channels = 3 if channels is None else channels
        n = len(ptrs)
        arr = (C.c_void_p * max(n, 1))(*ptrs)
        self._call(type(self)._ADD(self._h, self.added, n, arr, kind, channels))
        self.added += n


class BlendStream(_SourceStream):
    """A pano_blend_stream: the mosaic of pano_blend, fed window by window (LAZY_READ's memory contract).  A stream
    of rows (row0, row1) gives those rows of it and reads only the images needs() reports."""
    _NAME = "blend stream"
    _ADD = LIB.pano_blend_stream_add
    _FREE = LIB.pano_blend_stream_free
    _NULL_OK = True      # add() takes None for an image needs() reports False: passed as a null source

    def __init__(self, eng, handle, shapes, out_w, out_h, rows=None):
        super().__init__(eng, handle, shapes)
        self.out_w, self.out_h = out_w, out_h
        self.rows = tuple(rows) if rows is not None else (0, out_h)

    def needs(self):
        """bool per image: whether the stream reads its source (pano_blend_stream_needs)."""
        flags = np.zeros(max(len(self.shapes), 1), np.uint8)
        self._call(LIB.pano_blend_stream_needs(self._h, flags.ctypes.data))
        return flags[:len(self.shapes)].astype(bool)

    def finish(self):
        out = np.empty((self.rows[1] - self.rows[0], self.out_w, 3), np.float32)
        self._call(LIB.pano_blend_stream_finish(self._h, _f(out)))
        return out

    def finish_dev(self, d_out):
        self._call(LIB.pano_blend_stream_finish_dev(self._h, C.c_void_p(d_out or 0)))


SIZE_MAX = (1 << 64) - 1     # keep_bytes without a limit


def blend_sweep_plan(shapes, items, geom, bands, strip_rows, src_bytes, keep_bytes, params=None):
    """pano_blend_sweep_plan (no device needed): the strip schedule of a blend sweep.  Returns a dict with the
    strips × n bool arrays "reads", "uploads" and "kept" and the totals "n_uploads", "upload_bytes" and
    "retained_high"."""
    params = params or default_params()
    n = len(items)
    arr, g = Engine._blend_args([None] * n, shapes, items, geom)
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    S = -(-oh // strip_rows) if strip_rows > 0 else 0
    flags = [np.zeros(max(S * n, 1), np.uint8) for _ in range(3)]
    nb = (C.c_size_t * n)(*[int(b) for b in src_bytes])
    ns, nu = C.c_int(), C.c_longlong()
    ub, rh = C.c_ulonglong(), C.c_ulonglong()
    rc = LIB.pano_blend_sweep_plan(n, arr, C.byref(g), bands, C.byref(params), ow, oh, strip_rows, nb,
                                   min(int(keep_bytes), SIZE_MAX), C.byref(ns), *(f.ctypes.data for f in flags),
                                   C.byref(nu), C.byref(ub), C.byref(rh))
    if rc != 0:
        raise PanoError(rc, "blend sweep plan: bad argument")
    reads, uploads, kept = (f[:S * n].reshape(S, n).astype(bool) for f in flags)
    return {"reads": reads, "uploads": uploads, "kept": kept, "n_uploads": nu.value, "upload_bytes": ub.value,
            "retained_high": rh.value}


def blend_sweep_plan_cyl(shapes, items, geom, bands, corr_inv, strip_rows, src_bytes, keep_bytes, params=None):
    """pano_blend_sweep_plan_cyl (no device needed): blend_sweep_plan's schedule of a cylinder sweep whose
    perspective correction is corr_inv (3×3, row-major).  shapes / items / geom are the WARPED images'.  The dict
    also has "band", a strips × 2 int array of the mosaic rows [b0, b1) each strip blends."""
    params = params or default_params()
    n = len(items)
    arr, g = Engine._blend_args([None] * n, shapes, items, geom)
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    S = -(-oh // strip_rows) if strip_rows > 0 else 0
    flags = [np.zeros(max(S * n, 1), np.uint8) for _ in range(3)]
    band = np.zeros(max(2 * S, 1), np.int32)
    inv = np.ascontiguousarray(np.asarray(corr_inv, np.float64).reshape(9))
    nb = (C.c_size_t * n)(*[int(b) for b in src_bytes])
    ns, nu = C.c_int(), C.c_longlong()
    ub, rh = C.c_ulonglong(), C.c_ulonglong()
    rc = LIB.pano_blend_sweep_plan_cyl(n, arr, C.byref(g), bands, C.byref(params), ow, oh, _d(inv), strip_rows, nb,
                                       min(int(keep_bytes), SIZE_MAX), C.byref(ns), _i(band),
                                       *(f.ctypes.data for f in flags), C.byref(nu), C.byref(ub), C.byref(rh))
    if rc != 0:
        raise PanoError(rc, "cylinder blend sweep plan: bad argument")
    reads, uploads, kept = (f[:S * n].reshape(S, n).astype(bool) for f in flags)
    return {"band": band[:2 * S].reshape(S, 2), "reads": reads, "uploads": uploads, "kept": kept,
            "n_uploads": nu.value, "upload_bytes": ub.value, "retained_high": rh.value}


class BlendSweep(_Handle):
    """A pano_blend_sweep: the canvas's row strips top to bottom, each source handed over once while a later strip
    still reads it (within keep_bytes), then the cropped 8-bit mosaic.  next() gives the next strip and the images
    it wants, strip() takes them."""
    _FREE = LIB.pano_blend_sweep_free

    def __init__(self, eng, handle, n, out_w, out_h):
        self.eng, self._h, self.n, self.out_w, self.out_h = eng, handle, n, out_w, out_h

    def next(self):
        """(strip index or -1, bool array of the images strip() must be given)."""
        want = np.zeros(max(self.n, 1), np.uint8)
        r = LIB.pano_blend_sweep_next(self._h, want.ctypes.data)
        if r < -1:
            self._call(r)
        return r, want[:self.n].astype(bool)

    def strip(self, ptrs, formats, kind):
        """ptrs: n raw pointers (0 where next() did not ask), formats: n PANO_PIX_* codes (3 for f32 kinds)."""
        src = (C.c_void_p * max(self.n, 1))(*[int(q or 0) for q in ptrs])
        fm = (C.c_int * max(self.n, 1))(*[int(f) for f in formats])
        self._call(LIB.pano_blend_sweep_strip(self._h, src, fm, kind))

    def finish_dev(self, fmt, d_out):
        """Queues the mosaic's bytes in layout fmt into d_out; returns the rectangle {x0, y0, w, h}."""
        code = PIX_FORMATS.get(fmt, fmt) if isinstance(fmt, str) else fmt
        r = np.zeros(4, np.int32)
        self._call(LIB.pano_blend_sweep_finish_dev(self._h, int(code), C.c_void_p(d_out or 0), _i(r)))
        return r

    def stats(self):
        """(uploads, uploaded bytes, most bytes kept between two strips) so far."""
        u, b, r = C.c_longlong(), C.c_ulonglong(), C.c_ulonglong()
        self._call(LIB.pano_blend_sweep_stats(self._h, C.byref(u), C.byref(b), C.byref(r)))
        return u.value, b.value, r.value


class SiftStream(_SourceStream):
    """A pano_sift_stream: the featureset of sift_detect_batch (sift_detect_batch_rgb8 for uint8 sources), fed
    window by window (LAZY_READ's feature stage).  At most PANO_MAX_SIFT_BATCH images per add."""
    _NAME = "sift stream"
    _ADD = LIB.pano_sift_stream_add
    _FREE = LIB.pano_sift_stream_free

    def finish(self) -> FeatureSet:
        out = C.c_void_p()
        self._call(LIB.pano_sift_stream_finish(self._h, C.byref(out)))
        return FeatureSet(self.eng, out)


class CropScan(_Handle):
    """A pano_crop_scan: crop()'s rectangle of a mosaic that arrives in row strips (widths up to 80,000)."""
    _FREE = LIB.pano_crop_scan_free

    def __init__(self, eng, handle, w, h):
        self.eng, self._h, self.w, self.h = eng, handle, w, h

    def add_dev(self, d_strip, rows):
        """The next `rows` lines of the mosaic: a rows×w×3 f32 device buffer."""
        self._call(LIB.pano_crop_scan_add_dev(self._h, C.c_void_p(d_strip or 0), rows))

    def rect(self):
        """{x0, y0, width, height} once every line has been added."""
        r = np.zeros(4, np.int32)
        self._call(LIB.pano_crop_scan_rect(self._h, _i(r)))
        return r


def _lazy_windows(imgs, window, fmt):
    """The windows of sift_lazy / blend_lazy as (first, count, fmt), and every image's (h, w): window is an int or
    a list of sizes, fmt one value or a list with one per window (see pix_format)."""
    sizes = window if isinstance(window, (list, tuple)) else None
    wins, k = [], 0
    for q, n in enumerate(sizes if sizes is not None else iter(lambda: window, None)):
        if k >= len(imgs):
            break
        wins.append((k, n, fmt[q] if isinstance(fmt, (list, tuple)) else fmt))
        k += n
    shapes = [im.shape[:2] for im in imgs]
    for k0, n, f in wins:
        for i in range(k0, min(k0 + n, len(imgs))):
            if f is not None and imgs[i].dtype == np.uint8:
                shapes[i] = pix_format(imgs[i], f)[1:]
    return wins, shapes


class Engine:
    """One pano_ctx: a CUDA device + stream.  `stream` is a raw cudaStream_t
    (e.g. torch.cuda.current_stream().cuda_stream) or None."""

    def __init__(self, device: int = 0, stream: int | None = None):
        h = C.c_void_p()
        rc = LIB.pano_create(C.byref(h), device, C.c_void_p(stream) if stream else None)
        if rc != 0:
            raise PanoError(rc, LIB.pano_last_error(None).decode())
        self._h = h
        self.device = device

    # -- plumbing
    def _raise(self, rc):
        raise PanoError(rc, LIB.pano_last_error(self._h).decode())

    def _check(self, rc):
        if rc != 0:
            self._raise(rc)

    def close(self):
        if self._h:
            LIB.pano_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        self._check(LIB.pano_sync(self._h))

    @property
    def stream(self):
        return LIB.pano_stream(self._h)

    def trim(self):
        """Hand the freed device blocks this context keeps for reuse back to its pool."""
        self._check(LIB.pano_trim(self._h))

    def launch_count(self):
        return LIB.pano_launch_count(self._h)

    def mem_high_water(self, reset=False):
        """Peak bytes in use in this context's device pool since creation or the last reset."""
        v = C.c_size_t()
        self._check(LIB.pano_mem_high_water(self._h, C.byref(v), 1 if reset else 0))
        return v.value

    def match_last_exact_rows(self):
        return LIB.pano_match_last_exact_rows(self._h)

    def match_last_nominated_rows(self):
        return LIB.pano_match_last_nominated_rows(self._h)

    def profile(self, on: bool):
        self._check(LIB.pano_profile_enable(self._h, 1 if on else 0))

    def profile_reset(self):
        self._check(LIB.pano_profile_reset(self._h))

    def profile_read(self):
        cap = 64
        names = C.create_string_buffer(cap * 64)
        launches = (C.c_int * cap)()
        ms = (C.c_double * cap)()
        n = LIB.pano_profile_read(self._h, cap, names, launches, ms)
        out = {}
        for i in range(min(n, cap)):
            nm = names.raw[i * 64:(i + 1) * 64].split(b"\0", 1)[0].decode()
            out[nm] = (launches[i], ms[i])
        return out

    # -- device memory helpers (bench / tests)
    def dev_alloc(self, nbytes):
        p = C.c_void_p()
        self._check(LIB.pano_dev_alloc(self._h, nbytes, C.byref(p)))
        return p.value

    def dev_free(self, ptr):
        LIB.pano_dev_free(self._h, C.c_void_p(ptr))

    def dev_upload(self, ptr, arr):
        arr = np.ascontiguousarray(arr)
        self._check(LIB.pano_dev_upload(self._h, C.c_void_p(ptr), arr.ctypes.data_as(C.c_void_p), arr.nbytes))

    def dev_download(self, arr, ptr):
        assert arr.flags.c_contiguous
        self._check(LIB.pano_dev_download(self._h, arr.ctypes.data_as(C.c_void_p), C.c_void_p(ptr), arr.nbytes))

    def dev_upload_async(self, d_ptr, h_ptr, nbytes):
        self._check(LIB.pano_dev_upload_async(self._h, C.c_void_p(d_ptr), C.c_void_p(h_ptr), nbytes))

    def dev_download_async(self, h_ptr, d_ptr, nbytes):
        self._check(LIB.pano_dev_download_async(self._h, C.c_void_p(h_ptr), C.c_void_p(d_ptr), nbytes))

    @staticmethod
    def host_alloc(nbytes):
        p = C.c_void_p()
        if LIB.pano_host_alloc(nbytes, C.byref(p)) != 0:
            raise PanoError(-1, "pano_host_alloc failed")
        return p.value

    @staticmethod
    def host_free(ptr):
        LIB.pano_host_free(C.c_void_p(ptr))

    # -- events (cross-context ordering)
    def event_create(self):
        e = C.c_void_p()
        self._check(LIB.pano_event_create(self._h, C.byref(e)))
        return e

    def event_record(self, ev):
        self._check(LIB.pano_event_record(self._h, ev))

    def event_wait(self, ev):
        self._check(LIB.pano_event_wait(self._h, ev))

    @staticmethod
    def event_sync(ev):
        if LIB.pano_event_sync(ev) != 0:
            raise PanoError(-1, "pano_event_sync failed")

    @staticmethod
    def event_destroy(ev):
        LIB.pano_event_destroy(ev)

    # -- features
    def sift_detect_batch(self, imgs, params=None) -> FeatureSet:
        params = params or default_params()
        imgs = [np.ascontiguousarray(im, np.float32) for im in imgs]
        n = len(imgs)
        ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in imgs])
        ws = (C.c_int * n)(*[im.shape[1] for im in imgs])
        hs = (C.c_int * n)(*[im.shape[0] for im in imgs])
        out = C.c_void_p()
        self._check(LIB.pano_sift_detect_batch(self._h, n, ptrs, ws, hs, C.byref(params), C.byref(out)))
        return FeatureSet(self, out)

    def sift_detect_batch_ptr(self, ptrs, ws, hs, params=None, device=False) -> FeatureSet:
        """Raw-pointer variant (pinned host or device pointers), no numpy copies."""
        params = params or default_params()
        n = len(ptrs)
        cp = (C.c_void_p * n)(*ptrs)
        cw = (C.c_int * n)(*ws)
        ch = (C.c_int * n)(*hs)
        out = C.c_void_p()
        fn = LIB.pano_sift_detect_batch_dev if device else LIB.pano_sift_detect_batch
        self._check(fn(self._h, n, cp, cw, ch, C.byref(params), C.byref(out)))
        return FeatureSet(self, out)

    def sift_detect_batch_rgb8(self, pix, params=None, fmt=None) -> FeatureSet:
        """SIFT straight from decoded 8-bit pixels (numpy uint8 H×W, H×W×1 or H×W×3, read_img's input; with
        fmt="rgba" lodepng's H×W×4, with fmt="planar" CImg's 3×H×W; fmt may be a list, one per image): the
        features of sift_detect_batch on read_img's f32 images, without those images."""
        pix = [np.ascontiguousarray(x, np.uint8) for x in pix]
        fm = [pix_format(x, f) for x, f in zip(pix, _fmt_list(fmt, len(pix)))]
        return self.sift_detect_batch_rgb8_ptr([x.ctypes.data for x in pix], [f[2] for f in fm], [f[1] for f in fm],
                                               [f[0] for f in fm], params)

    def sift_detect_batch_rgb8_ptr(self, ptrs, ws, hs, channels, params=None, device=False) -> FeatureSet:
        """Raw-pointer variant: 8-bit images in host memory (pageable or pinned) or, with device=True, in device
        memory (valid until the first count query / download / match of the featureset); channels: one PANO_PIX_*
        code per image (1 or 3 for H×W×channels)."""
        params = params or default_params()
        n = len(ptrs)
        cp = (C.c_void_p * max(n, 1))(*ptrs)
        cw = (C.c_int * max(n, 1))(*ws)
        chh = (C.c_int * max(n, 1))(*hs)
        cc = (C.c_int * max(n, 1))(*channels)
        out = C.c_void_p()
        fn = LIB.pano_sift_detect_batch_rgb8_dev if device else LIB.pano_sift_detect_batch_rgb8
        self._check(fn(self._h, n, cp, cw, chh, cc, C.byref(params), C.byref(out)))
        return FeatureSet(self, out)

    def sift_detect(self, img, params=None):
        fs = self.sift_detect_batch([img], params)
        try:
            return fs.download(0)
        finally:
            fs.free()

    def sift_stream(self, shapes, params=None) -> SiftStream:
        """shapes: (h, w) per image.  Detects with `params` window by window; finish() returns the featureset."""
        params = params or default_params()
        n = len(shapes)
        ws = (C.c_int * max(n, 1))(*[int(s[1]) for s in shapes])
        hs = (C.c_int * max(n, 1))(*[int(s[0]) for s in shapes])
        h = C.c_void_p()
        self._check(LIB.pano_sift_stream_create(self._h, n, ws, hs, C.byref(params), C.byref(h)))
        return SiftStream(self, h, [tuple(s[:2]) for s in shapes])

    def sift_lazy(self, imgs, window=1, params=None, fmt=None) -> FeatureSet:
        """sift_detect_batch (uint8 sources: sift_detect_batch_rgb8) with the sources added `window` images at a
        time (an int, or a list of window sizes): numpy uint8 (H×W, H×W×1 or H×W×3) or float32 H×W×3 images.
        The images of one window share one channel count.  fmt: see pix_format; a list gives one per window."""
        wins, shapes = _lazy_windows(imgs, window, fmt)
        s = self.sift_stream(shapes, params)
        try:
            for k, q, f in wins:
                s.add(imgs[k:k + q], fmt=f)
            return s.finish()
        finally:
            s.close()

    def sift_trace(self, img, params=None) -> GpuSiftTrace:
        params = params or default_params()
        img = np.ascontiguousarray(img, np.float32)
        out = C.c_void_p()
        self._check(LIB.pano_sift_trace_run(self._h, _f(img), img.shape[1], img.shape[0], C.byref(params),
                                            C.byref(out)))
        return GpuSiftTrace(self, out)

    def featureset_upload(self, descs, coors=None) -> FeatureSet:
        descs = [np.ascontiguousarray(d, np.float32).reshape(-1, 128) for d in descs]
        n = len(descs)
        cnt = (C.c_int * n)(*[len(d) for d in descs])
        dp = (C.c_void_p * n)(*[d.ctypes.data for d in descs])
        cp = None
        if coors is not None:
            coors = [np.ascontiguousarray(c, np.float64).reshape(-1, 2) for c in coors]
            cp = (C.c_void_p * n)(*[c.ctypes.data for c in coors])
        out = C.c_void_p()
        self._check(LIB.pano_featureset_upload(self._h, n, cnt, dp, cp, C.byref(out)))
        return FeatureSet(self, out)

    def featureset_import_dev(self, counts, d_descs, d_coors=None) -> FeatureSet:
        """Featureset from device pointers (stream-ordered, no host sync)."""
        n = len(counts)
        cnt = (C.c_int * n)(*counts)
        dp = (C.c_void_p * n)(*d_descs)
        cp = (C.c_void_p * n)(*d_coors) if d_coors is not None else None
        out = C.c_void_p()
        self._check(LIB.pano_featureset_import_dev(self._h, n, cnt, dp, cp, C.byref(out)))
        return FeatureSet(self, out)

    def blend_rows_dev(self, ptrs, shapes, items, geom, d_out_rows, out_w, out_h, row0, row1, bands=0, params=None):
        """Rows [row0, row1) of the mosaic into a (row1-row0)×out_w×3 device buffer."""
        params = params or default_params()
        arr, g = self._blend_args(ptrs, shapes, items, geom)
        self._check(LIB.pano_blend_rows_dev(self._h, len(ptrs), arr, C.byref(g), bands, C.byref(params),
                                            C.c_void_p(d_out_rows), out_w, out_h, row0, row1))

    def blend_rows_rgb8_dev(self, d_pix, channels, shapes, items, geom, d_out_rows, out_w, out_h, row0, row1, bands=0,
                            params=None):
        """blend_rows_dev from device h×w×channels u8 sources (channels 1 or 3 per image): rows [row0, row1) of
        blend_rgb8_dev's mosaic.  Sources of images that do not reach the strip are never read."""
        params = params or default_params()
        n = len(d_pix)
        arr, g = self._blend_args([None] * n, shapes, items, geom)
        src = (C.c_void_p * max(n, 1))(*d_pix)
        ch = (C.c_int * max(n, 1))(*channels)
        self._check(LIB.pano_blend_rows_rgb8_dev(self._h, n, arr, src, ch, C.byref(g), bands, C.byref(params),
                                                 C.c_void_p(d_out_rows), out_w, out_h, row0, row1))

    # -- matching
    def match_pairs(self, fs: FeatureSet, pairs, params=None, shard=(0, 1)):
        """shard=(s, S): decide only share s of S of every pair's smaller set (row-sharded multi-GPU
        match); the shares' lists concatenated in shard order are the unsharded lists."""
        params = params or default_params()
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        m = PanoMatches()
        self._check(LIB.pano_match_pairs_shard(self._h, fs._h, len(pairs), _i(pairs), C.byref(params), int(shard[0]),
                                               int(shard[1]), C.byref(m)))
        n = m.n_pairs
        offs = np.ctypeslib.as_array(m.offset, shape=(n + 1,)).copy() if n else np.zeros(1, np.int32)
        total = int(offs[n]) if n else 0
        idx = (np.ctypeslib.as_array(m.idx, shape=(2 * total,)).reshape(-1, 2).copy() if total
               else np.zeros((0, 2), np.int32))
        LIB.pano_matches_free(C.byref(m))
        return [idx[offs[k]:offs[k + 1]] for k in range(n)]

    def match_pairs_dev(self, fs: FeatureSet, pairs, params=None, shard=(0, 1)) -> int:
        params = params or default_params()
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        tot = C.c_int()
        self._check(LIB.pano_match_pairs_dev_shard(self._h, fs._h, len(pairs), _i(pairs), C.byref(params), int(shard[0]),
                                                   int(shard[1]), C.byref(tot)))
        return tot.value

    def match_bruteforce(self, a, b, params=None):
        params = params or default_params()
        a = np.ascontiguousarray(a, np.float32).reshape(-1, 128)
        b = np.ascontiguousarray(b, np.float32).reshape(-1, 128)
        pairs = np.zeros((max(1, min(len(a), len(b))), 2), np.int32)
        n = C.c_int()
        self._check(LIB.pano_match_bruteforce(self._h, _f(a), len(a), _f(b), len(b), C.byref(params),
                                              _i(pairs), C.byref(n)))
        return pairs[:n.value].copy()

    # -- RANSAC inlier scoring
    def ransac_score_pairs(self, pairs):
        """pairs: list of (kp1_xy [n,2] f64, kp2_xy [n,2] f64, homos [m,9] f64, inlier_thres).
        Returns per pair (best_hyp, best_count, hyp_counts int32[m], inlier_flags uint8[n])."""
        n = len(pairs)
        arr = (PanoRansacPair * max(n, 1))()
        keep, counts, flags = [], [], []
        for k, (a, b, h, thr) in enumerate(pairs):
            a = np.ascontiguousarray(a, np.float64).reshape(-1, 2)
            b = np.ascontiguousarray(b, np.float64).reshape(-1, 2)
            h = np.ascontiguousarray(h, np.float64).reshape(-1, 9)
            keep.append((a, b, h))
            arr[k].n_match, arr[k].kp1_xy, arr[k].kp2_xy = len(a), a.ctypes.data, b.ctypes.data
            arr[k].n_hyp, arr[k].homos, arr[k].inlier_thres = len(h), h.ctypes.data, thr
            counts.append(np.zeros(max(len(h), 1), np.int32))
            flags.append(np.zeros(max(len(a), 1), np.uint8))
        best, bcnt = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        cp = (C.c_void_p * max(n, 1))(*[c.ctypes.data for c in counts])
        fp = (C.c_void_p * max(n, 1))(*[f.ctypes.data for f in flags])
        self._check(LIB.pano_ransac_score_pairs(self._h, n, arr, _i(best), _i(bcnt), cp, fp))
        return [(int(best[k]), int(bcnt[k]), counts[k][:len(keep[k][2])], flags[k][:len(keep[k][0])]) for k in range(n)]

    # -- bundle-adjustment Jacobian assembly
    def ba_jacobian(self, n_cam, pairs, pts_to, want_rows=True):
        """pairs: list of (from_slot, to_slot, n_match, mats [13, 9] f64) in match order; pts_to: [n_match_total, 2].
        Returns (j_rows [n_match_total, 24] or None, jtj [6 n_cam, 6 n_cam])."""
        n = len(pairs)
        arr = (PanoBaPair * max(n, 1))()
        begin = 0
        for k, (f, t, nm, mats) in enumerate(pairs):
            arr[k].from_, arr[k].to, arr[k].match_begin, arr[k].n_match = f, t, begin, nm
            C.memmove(arr[k].m, np.ascontiguousarray(mats, np.float64).ctypes.data, 13 * 9 * 8)
            begin += nm
        pts_to = np.ascontiguousarray(pts_to, np.float64).reshape(-1, 2)
        assert len(pts_to) == begin
        rows = np.zeros((max(begin, 1), 24), np.float64) if want_rows else None
        jtj = np.full((6 * n_cam, 6 * n_cam), np.nan, np.float64)
        self._check(LIB.pano_ba_jacobian(self._h, n_cam, n, arr, _d(pts_to), _d(rows) if want_rows else None, _d(jtj)))
        return (rows[:begin] if want_rows else None), jtj

    def ba_session(self, n_cam, pairs, pts) -> BaSession:
        """pairs: list of (from_slot, to_slot, n_match) in match order; pts: [n_match_total, 4] =
        p.first.x, p.first.y, p.second.x, p.second.y of MatchInfo::match (to, then from)."""
        n = len(pairs)
        arr = (PanoBaLink * max(n, 1))()
        begin = 0
        for k, (f, t, nm) in enumerate(pairs):
            arr[k].from_, arr[k].to, arr[k].match_begin, arr[k].n_match = f, t, begin, nm
            begin += nm
        pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 4)
        if len(pts) != begin:
            raise PanoError(-2, f"ba session: {len(pts)} coordinate rows for {begin} matches")
        h = C.c_void_p()
        self._check(LIB.pano_ba_session_create(self._h, n_cam, n, arr, _d(pts) if len(pts) else None, C.byref(h)))
        return BaSession(self, h, n_cam, n, begin)

    # -- cylinder warp
    @staticmethod
    def cyl_warp_shape(w, h, h_factor=1.0, params=None):
        params = params or default_params()
        ow, oh, ox, oy = C.c_int(), C.c_int(), C.c_double(), C.c_double()
        rc = LIB.pano_cyl_warp_shape(w, h, h_factor, C.byref(params), C.byref(ow), C.byref(oh), C.byref(ox),
                                     C.byref(oy))
        if rc:
            raise PanoError(rc, "pano_cyl_warp_shape")
        return ow.value, oh.value, ox.value, oy.value

    def cyl_warp(self, img, kpts=None, h_factor=1.0, params=None):
        params = params or default_params()
        img = np.ascontiguousarray(img, np.float32)
        ow, oh, _, _ = self.cyl_warp_shape(img.shape[1], img.shape[0], h_factor, params)
        out = np.empty((oh, ow, 3), np.float32)
        k = np.ascontiguousarray(kpts if kpts is not None else np.zeros((0, 2)), np.float64).copy()
        self._check(LIB.pano_cyl_warp(self._h, _f(img), img.shape[1], img.shape[0], h_factor, C.byref(params),
                                      _f(out), ow, oh, _d(k), len(k)))
        return out, k

    def _cyl_jobs(self, src_ptrs, shapes, dst_ptrs, kpts, h_factor, params):
        n = len(src_ptrs)
        arr = (PanoCylJob * max(n, 1))()
        for k in range(n):
            h, w = shapes[k]
            ow, oh, _, _ = self.cyl_warp_shape(w, h, h_factor, params)
            arr[k].d_rgb_hwc, arr[k].w, arr[k].h = src_ptrs[k], w, h
            arr[k].d_out_hwc, arr[k].out_w, arr[k].out_h = dst_ptrs[k], ow, oh
            if kpts is not None and kpts[k] is not None and len(kpts[k]):
                assert kpts[k].dtype == np.float64 and kpts[k].flags["C_CONTIGUOUS"]
                arr[k].kpts_xy, arr[k].n_kpts = kpts[k].ctypes.data, len(kpts[k])
        return arr

    def cyl_warp_batch_dev(self, src_ptrs, shapes, dst_ptrs, kpts=None, h_factor=1.0, params=None):
        """Device pointers in, device pointers out (out sizes from cyl_warp_shape), asynchronous; kpts: optional
        list of [n, 2] float64 arrays rewritten in place."""
        params = params or default_params()
        arr = self._cyl_jobs(src_ptrs, shapes, dst_ptrs, kpts, h_factor, params)
        self._check(LIB.pano_cyl_warp_batch_dev(self._h, len(src_ptrs), arr, h_factor, C.byref(params)))

    def cyl_warp_batch_rgb8_dev(self, src_ptrs, channels, shapes, dst_ptrs, kpts=None, h_factor=1.0, params=None):
        """cyl_warp_batch_dev from device h×w×channels u8 sources (channels 1 or 3 per image): the warp of
        cyl_warp_batch_dev on read_img's f32 images of the same pixels."""
        params = params or default_params()
        n = len(src_ptrs)
        arr = self._cyl_jobs([None] * n, shapes, dst_ptrs, kpts, h_factor, params)
        src = (C.c_void_p * max(n, 1))(*src_ptrs)
        ch = (C.c_int * max(n, 1))(*channels)
        self._check(LIB.pano_cyl_warp_batch_rgb8_dev(self._h, n, arr, src, ch, h_factor, C.byref(params)))

    # -- blend
    @staticmethod
    def _blend_args(imgs_or_ptrs, shapes, items, geom):
        n = len(items)
        arr = (PanoBlendImage * n)()
        for k in range(n):
            arr[k].rgb_hwc = imgs_or_ptrs[k]
            arr[k].h, arr[k].w = shapes[k]
            arr[k].x0, arr[k].y0, arr[k].x1, arr[k].y1 = items[k][:4]
            for q in range(9):
                arr[k].homo_inv[q] = items[k][4][q]
        g = PanoBlendGeom(projection=geom["projection"], res_x=geom["res_x"], res_y=geom["res_y"],
                          proj_min_x=geom["proj_min_x"], proj_min_y=geom["proj_min_y"])
        return arr, g

    def blend(self, imgs, items, geom, bands=0, params=None):
        """imgs: list of HxWx3 float32; items: (x0,y0,x1,y1,homo_inv[9]) per image."""
        params = params or default_params()
        imgs = [np.ascontiguousarray(im, np.float32) for im in imgs]
        arr, g = self._blend_args([im.ctypes.data for im in imgs], [im.shape[:2] for im in imgs], items, geom)
        ow, oh = C.c_int(), C.c_int()
        LIB.pano_blend_target_size(len(imgs), arr, C.byref(ow), C.byref(oh))
        out = np.empty((oh.value, ow.value, 3), np.float32)
        self._check(LIB.pano_blend(self._h, len(imgs), arr, C.byref(g), bands, C.byref(params), _f(out),
                                   ow.value, oh.value))
        return out

    def blend_dev(self, ptrs, shapes, items, geom, d_out, out_w, out_h, bands=0, params=None):
        params = params or default_params()
        arr, g = self._blend_args(ptrs, shapes, items, geom)
        self._check(LIB.pano_blend_dev(self._h, len(ptrs), arr, C.byref(g), bands, C.byref(params),
                                       C.c_void_p(d_out), out_w, out_h))

    def blend_rgb8_dev(self, d_pix, channels, shapes, items, geom, d_out, out_w, out_h, bands=0, params=None):
        """blend_dev from device h×w×channels u8 sources (channels 1 or 3 per image): the mosaic of blend_dev on
        read_img's f32 images of the same pixels."""
        params = params or default_params()
        n = len(d_pix)
        arr, g = self._blend_args([None] * n, shapes, items, geom)
        src = (C.c_void_p * max(n, 1))(*d_pix)
        ch = (C.c_int * max(n, 1))(*channels)
        self._check(LIB.pano_blend_rgb8_dev(self._h, n, arr, src, ch, C.byref(g), bands, C.byref(params),
                                            C.c_void_p(d_out), out_w, out_h))

    def blend_stream(self, shapes, items, geom, bands=0, params=None) -> BlendStream:
        """shapes: (h, w) per image; items / geom as for blend().  Allocates the canvas state."""
        params = params or default_params()
        arr, g = self._blend_args([None] * len(items), shapes, items, geom)
        ow, oh = C.c_int(), C.c_int()
        self._check(LIB.pano_blend_target_size(len(items), arr, C.byref(ow), C.byref(oh)))
        h = C.c_void_p()
        self._check(LIB.pano_blend_stream_create(self._h, len(items), arr, C.byref(g), bands, C.byref(params), ow.value,
                                                 oh.value, C.byref(h)))
        return BlendStream(self, h, shapes, ow.value, oh.value)

    def blend_stream_rows(self, shapes, items, geom, row0, row1, bands=0, params=None) -> BlendStream:
        """blend_stream for rows [row0, row1) of the canvas only: finish() gives those rows of the mosaic."""
        params = params or default_params()
        arr, g = self._blend_args([None] * len(items), shapes, items, geom)
        ow, oh = C.c_int(), C.c_int()
        self._check(LIB.pano_blend_target_size(len(items), arr, C.byref(ow), C.byref(oh)))
        h = C.c_void_p()
        self._check(LIB.pano_blend_stream_create_rows(self._h, len(items), arr, C.byref(g), bands, C.byref(params),
                                                      ow.value, oh.value, row0, row1, C.byref(h)))
        return BlendStream(self, h, shapes, ow.value, oh.value, (row0, row1))

    def blend_stream_cyl(self, src_shapes, items, geom, h_factor, bands=0, params=None) -> BlendStream:
        """blend_stream over cylinder mode's warped images, fed the UNWARPED sources: src_shapes are the sources'
        (h, w), items / geom those of the warped images (each of cyl_warp_shape's size).  add() takes the sources;
        finish() gives blend_dev's mosaic of the images cyl_warp_batch_dev warps from them."""
        params = params or default_params()
        n = len(items)
        shapes = []
        for h, w in src_shapes:
            try:
                ow, oh, _, _ = self.cyl_warp_shape(w, h, h_factor, params)
            except PanoError:
                ow, oh = 0, 0
            shapes.append((oh, ow))
        arr, g = self._blend_args([None] * n, shapes, items, geom)
        ow, oh = C.c_int(), C.c_int()
        self._check(LIB.pano_blend_target_size(n, arr, C.byref(ow), C.byref(oh)))
        sw = (C.c_int * max(n, 1))(*[int(s[1]) for s in src_shapes])
        sh = (C.c_int * max(n, 1))(*[int(s[0]) for s in src_shapes])
        h = C.c_void_p()
        self._check(LIB.pano_blend_stream_create_cyl(self._h, n, arr, sw, sh, h_factor, C.byref(g), bands,
                                                     C.byref(params), ow.value, oh.value, C.byref(h)))
        return BlendStream(self, h, src_shapes, ow.value, oh.value)

    def blend_sweep(self, shapes, items, geom, strip_rows, keep_bytes, bands=0, params=None, crop=True,
                    src_bytes=None) -> BlendSweep:
        """A blend sweep (pano_blend_sweep_create) of strips of strip_rows canvas rows, keeping at most keep_bytes of
        sources (SIZE_MAX: no limit) between strips; src_bytes: each source's bytes (None: h·w·3)."""
        params = params or default_params()
        n = len(items)
        arr, g = self._blend_args([None] * n, shapes, items, geom)
        ow, oh = C.c_int(), C.c_int()
        self._check(LIB.pano_blend_target_size(n, arr, C.byref(ow), C.byref(oh)))
        nb = (C.c_size_t * n)(*[int(b) for b in src_bytes]) if src_bytes is not None else None
        h = C.c_void_p()
        self._check(LIB.pano_blend_sweep_create(self._h, n, arr, C.byref(g), bands, C.byref(params), ow.value, oh.value,
                                                strip_rows, nb, min(int(keep_bytes), SIZE_MAX), 1 if crop else 0,
                                                C.byref(h)))
        return BlendSweep(self, h, n, ow.value, oh.value)

    def blend_sweep_cyl(self, src_shapes, items, geom, h_factor, corr_inv, strip_rows, keep_bytes, bands=0,
                        params=None, crop=True, src_bytes=None) -> BlendSweep:
        """A cylinder sweep (pano_blend_sweep_create_cyl): write_rgb(crop(perspective_correction(mosaic))) of the
        mosaic blend_stream_cyl gives, strip by strip.  src_shapes: the UNWARPED sources' (h, w); items / geom: the
        warped images'; corr_inv: perspective_correction's inv (3×3, row-major); src_bytes: each source's bytes
        (None: h·w·3).  strip() takes the unwarped sources."""
        params = params or default_params()
        n = len(items)
        shapes = []
        for h, w in src_shapes:
            try:
                ow, oh, _, _ = self.cyl_warp_shape(w, h, h_factor, params)
            except PanoError:
                ow, oh = 0, 0
            shapes.append((oh, ow))
        arr, g = self._blend_args([None] * n, shapes, items, geom)
        ow, oh = C.c_int(), C.c_int()
        self._check(LIB.pano_blend_target_size(n, arr, C.byref(ow), C.byref(oh)))
        sw = (C.c_int * max(n, 1))(*[int(s[1]) for s in src_shapes])
        sh = (C.c_int * max(n, 1))(*[int(s[0]) for s in src_shapes])
        inv = np.ascontiguousarray(np.asarray(corr_inv, np.float64).reshape(9))
        nb = (C.c_size_t * n)(*[int(b) for b in src_bytes]) if src_bytes is not None else None
        h = C.c_void_p()
        self._check(LIB.pano_blend_sweep_create_cyl(self._h, n, arr, sw, sh, h_factor, C.byref(g), bands,
                                                    C.byref(params), ow.value, oh.value, _d(inv), strip_rows, nb,
                                                    min(int(keep_bytes), SIZE_MAX), 1 if crop else 0, C.byref(h)))
        return BlendSweep(self, h, n, ow.value, oh.value)

    def blend_lazy(self, imgs, items, geom, bands=0, params=None, window=1, fmt=None):
        """blend() with the sources added `window` images at a time (an int, or a list of window sizes):
        numpy uint8 (read_img's input: H×W, H×W×1 or H×W×3) or float32 H×W×3 images.  fmt: see pix_format; a
        list gives one per window."""
        wins, shapes = _lazy_windows(imgs, window, fmt)
        s = self.blend_stream(shapes, items, geom, bands, params)
        try:
            for k, q, f in wins:
                s.add(imgs[k:k + q], fmt=f)
            return s.finish()
        finally:
            s.close()

    # -- little planet (main.cc:294-331)
    PLANET_SIZE = 1000                 # PANO_PLANET_SIZE, main.cc:297

    def planet(self, img):
        """img: H×W×3 float32 mosaic (-1 = Color::NO) -> (1000, 1000, 3) float32, -1 where nothing maps."""
        img = np.ascontiguousarray(img, np.float32)
        if img.ndim != 3 or img.shape[2] != 3:
            raise PanoError(-2, f"planet: expected an H×W×3 image, got shape {img.shape}")
        out = np.empty((self.PLANET_SIZE, self.PLANET_SIZE, 3), np.float32)
        self._check(LIB.pano_planet(self._h, _f(img), img.shape[1], img.shape[0], _f(out)))
        return out

    def planet_dev(self, d_src, w, h, d_out):
        """Device pointers in and out (d_out: 1000×1000×3 f32), asynchronous on the context's stream."""
        self._check(LIB.pano_planet_dev(self._h, C.c_void_p(d_src or 0), w, h, C.c_void_p(d_out or 0)))

    def planet_pix8(self, pix, fmt=None):
        """planet() of a decoded 8-bit image (uint8 H×W, H×W×1 or H×W×3; lodepng's H×W×4 with fmt="rgba", CImg's
        3×H×W with fmt="planar"; see pix_format), uploaded as it is -> (1000, 1000, 3) float32: the bits of
        planet(read_img_rgb8(pix, fmt)) without that f32 image."""
        pix = np.ascontiguousarray(pix, np.uint8)
        code, h, w = pix_format(pix, fmt)
        out = np.empty((self.PLANET_SIZE, self.PLANET_SIZE, 3), np.float32)
        self._check(LIB.pano_planet_pix8(self._h, C.c_void_p(pix.ctypes.data), code, w, h, _f(out)))
        return out

    def planet_pix8_dev(self, d_pix, fmt, w, h, d_out):
        """Device pointers in and out (d_out: 1000×1000×3 f32), asynchronous on the context's stream; fmt is a
        PANO_PIX_* code or "grey" / "rgb" / "rgba" / "planar"."""
        code = PIX_FORMATS.get(fmt, fmt) if isinstance(fmt, str) else fmt
        self._check(LIB.pano_planet_pix8_dev(self._h, C.c_void_p(d_pix or 0), int(code), w, h, C.c_void_p(d_out or 0)))

    # ---- 8-bit boundary: read_img / crop / write_rgb formats (device pointers)
    def rgb8_to_mat32f_batch_dev(self, d_pix, ws, hs, channels, d_out):
        """u8 -> f32 for n images in one launch (read_img's conversion, imgio.cc:75-88)."""
        n = len(d_pix)
        src = (C.c_void_p * n)(*d_pix)
        dst = (C.c_void_p * n)(*d_out)
        self._check(LIB.pano_rgb8_to_mat32f_batch_dev(self._h, n, src, (C.c_int * n)(*ws), (C.c_int * n)(*hs),
                                                      (C.c_int * n)(*channels), dst))

    def rgb8_to_mat32f_dev(self, d_pix, w, h, channels, d_out):
        self._check(LIB.pano_rgb8_to_mat32f_dev(self._h, C.c_void_p(d_pix), w, h, channels, C.c_void_p(d_out)))

    def crop_rect_dev(self, d_mat, w, h, d_rect):
        """crop()'s rectangle (imgproc.cc:200-235) into device int[4] {x0,y0,w,h}."""
        self._check(LIB.pano_crop_rect_dev(self._h, C.c_void_p(d_mat), w, h, C.c_void_p(d_rect)))

    def mat32f_to_rgb8_dev(self, d_mat, w, h, d_rect, d_out):
        """write_rgb's conversion (imgio.cc:98-113) of the rectangle d_rect (0/None = whole image)."""
        self._check(LIB.pano_mat32f_to_rgb8_dev(self._h, C.c_void_p(d_mat), w, h, C.c_void_p(d_rect or 0),
                                                C.c_void_p(d_out)))

    def crop_scan(self, w, h) -> CropScan:
        h_ = C.c_void_p()
        self._check(LIB.pano_crop_scan_create(self._h, w, h, C.byref(h_)))
        return CropScan(self, h_, w, h)

    def rgb8_crop_to_pix8_dev(self, d_rgb8, w, h, d_rect, fmt, d_out):
        """mat32f_to_pix8_dev's bytes from the h×w×3 u8 mosaic mat32f_to_rgb8_dev wrote without a rect."""
        code = PIX_FORMATS.get(fmt, fmt) if isinstance(fmt, str) else fmt
        self._check(LIB.pano_rgb8_crop_to_pix8_dev(self._h, C.c_void_p(d_rgb8), w, h, C.c_void_p(d_rect or 0),
                                                   int(code), C.c_void_p(d_out)))

    def mat32f_to_pix8_dev(self, d_mat, w, h, d_rect, fmt, d_out):
        """The same conversion in an encoder's layout: fmt is a PANO_PIX_* code or "rgb" / "rgba" (write_png's
        buffer, alpha 255) / "planar" (write_rgb's CImg planes), packed to the rectangle's size."""
        code = PIX_FORMATS.get(fmt, fmt) if isinstance(fmt, str) else fmt
        self._check(LIB.pano_mat32f_to_pix8_dev(self._h, C.c_void_p(d_mat), w, h, C.c_void_p(d_rect or 0), int(code),
                                                C.c_void_p(d_out)))

    # numpy conveniences for tests
    def read_img_rgb8(self, pix, fmt=None):
        pix = np.ascontiguousarray(pix, np.uint8)
        ch, h, w = pix_format(pix, fmt)
        d_in = self.dev_alloc(max(pix.nbytes, 256))
        d_out = self.dev_alloc(h * w * 12)
        out = np.empty((h, w, 3), np.float32)
        try:
            self.dev_upload(d_in, pix)
            self.rgb8_to_mat32f_dev(d_in, w, h, ch, d_out)
            self.dev_download(out, d_out)
        finally:
            self.dev_free(d_in)
            self.dev_free(d_out)
        return out

    def crop_write_rgb8(self, mat, crop=True):
        """Returns (rect or None, 8-bit pixels of the (cropped) mosaic)."""
        mat = np.ascontiguousarray(mat, np.float32)
        h, w = mat.shape[:2]
        d_mat = self.dev_alloc(mat.nbytes)
        d_rect = self.dev_alloc(256)
        d_out = self.dev_alloc(max(h * w * 3, 256))
        rect = np.zeros(4, np.int32)
        out = np.empty(h * w * 3, np.uint8)
        try:
            self.dev_upload(d_mat, mat)
            if crop:
                self.crop_rect_dev(d_mat, w, h, d_rect)
            self.mat32f_to_rgb8_dev(d_mat, w, h, d_rect if crop else 0, d_out)
            self.dev_download(out, d_out)
            if crop:
                self.dev_download(rect, d_rect)
        finally:
            for p_ in (d_mat, d_rect, d_out):
                self.dev_free(p_)
        if not crop:
            return None, out.reshape(h, w, 3)
        cw, ch = int(rect[2]), int(rect[3])
        return rect, out[:cw * ch * 3].reshape(ch, cw, 3).copy()

    def crop_write_pix8(self, mat, crop=True, fmt="rgb"):
        """crop_write_rgb8 with the pixels in layout fmt: "rgb" (ch×cw×3), "rgba" (ch×cw×4, alpha 255) or
        "planar" (3×ch×cw)."""
        mat = np.ascontiguousarray(mat, np.float32)
        h, w = mat.shape[:2]
        code = PIX_FORMATS[fmt]
        bpp = 4 if code == PIX_RGBA else 3
        d_mat = self.dev_alloc(mat.nbytes)
        d_rect = self.dev_alloc(256)
        d_out = self.dev_alloc(max(h * w * bpp, 256))
        rect = np.zeros(4, np.int32)
        out = np.empty(h * w * bpp, np.uint8)
        try:
            self.dev_upload(d_mat, mat)
            if crop:
                self.crop_rect_dev(d_mat, w, h, d_rect)
            self.mat32f_to_pix8_dev(d_mat, w, h, d_rect if crop else 0, code, d_out)
            self.dev_download(out, d_out)
            if crop:
                self.dev_download(rect, d_rect)
        finally:
            for p_ in (d_mat, d_rect, d_out):
                self.dev_free(p_)
        cw, ch = (int(rect[2]), int(rect[3])) if crop else (w, h)
        px = out[:cw * ch * bpp]
        px = px.reshape(3, ch, cw) if code == PIX_RGB_PLANAR else px.reshape(ch, cw, bpp)
        return (rect if crop else None), px.copy()
