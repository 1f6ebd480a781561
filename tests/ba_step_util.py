"""Checker wrappers and cases for one LM iteration of bundle adjustment (calcError, update_stats and
b = J^T * err_vec, incremental_bundle_adjuster.cc:171-238): orc_ba_error / orc_ba_jtr (the plain-C
restatement, oracle/liboracle_ba_step.so) and ref_ba_error / ref_ba_jtr (the reference's own TU,
oracle/_ref/libopenpano_ref_ba_step.so), both built by oracle/ba_step.mk."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

from openpano_b200._abi import PanoBaPair
from tests.ba_util import rodrigues

_dp = C.POINTER(C.c_double)
ROOT = Path(__file__).resolve().parent.parent
ORC_SO = ROOT / "oracle" / "liboracle_ba_step.so"
REF_SO = ROOT / "oracle" / "_ref" / "libopenpano_ref_ba_step.so"
_libs = {}


def _lib(path):
    if path not in _libs:
        if path == ORC_SO and not path.exists():
            subprocess.check_call(["make", "-s", "-C", str(ROOT / "oracle"), "-f", "ba_step.mk", "oracle"])
        _libs[path] = C.CDLL(str(path))
    return _libs[path]


def have_ref():
    return REF_SO.exists()


def _d(a):
    return a.ctypes.data_as(_dp)


def _pairs(pairs):
    arr = (PanoBaPair * max(len(pairs), 1))()
    begin = 0
    for k, (f, t, nm) in enumerate(pairs):
        arr[k].from_, arr[k].to, arr[k].match_begin, arr[k].n_match = f, t, begin, nm
        begin += nm
    return arr, begin


def rejected_cams(cams, seed):
    """A perturbed copy of the cameras: the `new_state` of an LM step that optimize() rejects (:146-153)."""
    rng = np.random.RandomState(seed)
    out = np.array(cams, np.float64).reshape(-1, 12).copy()
    for c in out:
        c[0] += 5.0 * rng.randn()
        c[1:3] += rng.randn(2)
        c[3:] = (c[3:].reshape(3, 3) @ rodrigues(0.002 * rng.randn(3))).reshape(-1)
    return out


def orc_error(pairs, hto, pts):
    """-> (residuals [2 n_match], avg, max)."""
    arr, total = _pairs(pairs)
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 4)
    hto = np.ascontiguousarray(hto, np.float64).reshape(-1)
    assert total == len(pts) and hto.size == 9 * len(pairs)
    res = np.zeros(max(2 * total, 1), np.float64)
    avg, mx = C.c_double(), C.c_double()
    fn = _lib(ORC_SO).orc_ba_error
    fn.argtypes = [C.c_int, C.POINTER(PanoBaPair), _dp, _dp, _dp, _dp, _dp]
    assert fn(len(pairs), arr, _d(hto), _d(pts), _d(res), C.byref(avg), C.byref(mx)) == 0
    return res[:2 * total], avg.value, mx.value


def orc_jtr(n_cam, pairs, rows, residuals):
    """b = J^T * residuals from the compact rows of orc_ba_jacobian -> [6 n_cam]."""
    arr, total = _pairs(pairs)
    rows = np.ascontiguousarray(rows, np.float64).reshape(-1, 24)
    residuals = np.ascontiguousarray(residuals, np.float64).reshape(-1)
    assert len(rows) == total and residuals.size == 2 * total
    b = np.full(6 * n_cam, np.nan, np.float64)
    fn = _lib(ORC_SO).orc_ba_jtr
    fn.argtypes = [C.c_int, C.c_int, C.POINTER(PanoBaPair), _dp, _dp, _dp]
    assert fn(n_cam, len(pairs), arr, _d(rows) if total else None, _d(residuals) if total else None, _d(b)) == 0
    return b


def ref_error(cams, pairs, pts):
    """The reference's own calcError(state) -> (residuals, avg, max, hto [n_pair, 9] made by its operations)."""
    cams = np.ascontiguousarray(cams, np.float64).reshape(-1, 12)
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 4)
    arr, total = _pairs(pairs)
    assert total == len(pts)
    res = np.zeros(max(2 * total, 1), np.float64)
    hto = np.zeros((max(len(pairs), 1), 9), np.float64)
    avg, mx = C.c_double(), C.c_double()
    fn = _lib(REF_SO).ref_ba_error
    fn.argtypes = [C.c_int, _dp, C.c_int, C.POINTER(PanoBaPair), _dp, _dp, _dp, _dp, _dp]
    assert fn(len(cams), _d(cams), len(pairs), arr, _d(pts), _d(res), C.byref(avg), C.byref(mx), _d(hto)) == 0
    return res[:2 * total], avg.value, mx.value, hto[:len(pairs)]


def ref_jtr(cams, pairs, pts, residuals):
    """The reference's calcJacobianSymbolic(state), then J.transpose() * Map(residuals) -> b [6 n_cam]."""
    cams = np.ascontiguousarray(cams, np.float64).reshape(-1, 12)
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 4)
    residuals = np.ascontiguousarray(residuals, np.float64).reshape(-1)
    arr, total = _pairs(pairs)
    assert total == len(pts) and residuals.size == 2 * total
    b = np.full(6 * len(cams), np.nan, np.float64)
    fn = _lib(REF_SO).ref_ba_jtr
    fn.argtypes = [C.c_int, _dp, C.c_int, C.POINTER(PanoBaPair), _dp, _dp, _dp]
    assert fn(len(cams), _d(cams), len(pairs), arr, _d(pts), _d(residuals), _d(b)) == 0
    return b
