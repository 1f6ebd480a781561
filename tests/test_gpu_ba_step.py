"""GPU: one LM iteration's per-point work of bundle adjustment on a device-resident session
(pano_ba_session: calcError + update_stats, J, J^T J and b = J^T * err_vec, incremental_bundle_adjuster.cc:
171-238) against the golden fixture made by the reference's own TU and against the plain-C restatement,
bit for bit, up to the size the reference's comment names ("J.rows() could reach 700000")."""
import ctypes as C
import os
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import ba_step_util as bs
from tests import golden_util as gu
from tests.ba_util import ba_case, numpy_pair_mats

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "ba_step_test"


def _want(orc, n_cam, pairs, mats, hto, pts, hto_b=None):
    """Restatement: residuals, avg, max at hto; rows and J^T J at mats; b with the residuals at hto_b (or hto)."""
    res, avg, mx = bs.orc_error(pairs, hto, pts)
    rows, jtj = orc.ba_jacobian(n_cam, pairs, mats, pts[:, :2])
    res_b = res if hto_b is None else bs.orc_error(pairs, hto_b, pts)[0]
    return res, avg, mx, rows, jtj, bs.orc_jtr(n_cam, pairs, rows, res_b)


def same_b(b, want):
    """Bit for bit, except that a NaN only has to be a NaN: the default NaN of x86 and of the GPU need not share
    a sign bit."""
    nan = np.isnan(want)
    return np.array_equal(np.isnan(b), nan) and gu.same_bits(b[~nan], want[~nan])


def test_ba_step_matches_golden(engine):
    """The reference's own calcError and J^T * err_vec (tests/golden/ba_step_5cams.npz), at a state and after a
    rejected step; J and J^T J against tests/golden/ba_5cams.npz (the reference's calcJacobianSymbolic)."""
    g, gj = gu.load("ba_step_5cams.npz"), gu.load("ba_5cams.npz")
    cams, pairs, pts = ba_case(5, 40, 5, extra_pairs=3)
    assert str(g["input_sha"]) == gu.sha(cams, np.array(pairs), pts)
    s = engine.ba_session(5, pairs, pts)
    try:
        for sfx in ("", "_rejected"):
            avg, mx, res = s.error(g["hto" + sfx])
            assert gu.same_bits(res, g["residuals" + sfx])
            assert gu.same_bits(np.float64(avg), g["avg" + sfx]) and gu.same_bits(np.float64(mx), g["max" + sfx])
            jtj, b, rows = s.normal_equations(g["mats"], want_rows=True)
            assert gu.same_bits(b, g["b" + sfx])
            assert gu.same_bits(rows, gj["rows"]) and gu.same_bits(jtj, gj["jtj"])
    finally:
        s.close()


@pytest.mark.parametrize("n_cam,per_pair,seed,extra", [(3, 1, 3, 0), (38, 400, 7, 60), (24, 9000, 8, 16)])
def test_ba_step_bit_exact(engine, orc, n_cam, per_pair, seed, extra):
    cams, pairs, pts = ba_case(n_cam, per_pair, seed, extra_pairs=extra)
    mats = numpy_pair_mats(cams, pairs)        # any matrices are valid inputs of the per-point code
    hto = mats[:, 0]
    w_res, w_avg, w_max, w_rows, w_jtj, w_b = _want(orc, n_cam, pairs, mats, hto, pts)
    s = engine.ba_session(n_cam, pairs, pts)
    try:
        avg, mx, res = s.error(hto)
        assert gu.same_bits(res, w_res)
        assert gu.same_bits(np.float64(avg), np.float64(w_avg)) and gu.same_bits(np.float64(mx), np.float64(w_max))
        jtj, b, rows = s.normal_equations(mats, want_rows=True)
        assert gu.same_bits(rows, w_rows) and gu.same_bits(jtj, w_jtj) and gu.same_bits(b, w_b)
        # the same J / J^T J as pano_ba_jacobian on the same input; J^T J and b without the rows coming back
        rows2, jtj2 = engine.ba_jacobian(n_cam, [(f, t, n, m) for (f, t, n), m in zip(pairs, mats)], pts[:, :2])
        assert gu.same_bits(rows, rows2) and gu.same_bits(jtj, jtj2)
        jtj3, b3, none = s.normal_equations(mats)
        assert none is None and gu.same_bits(jtj3, w_jtj) and gu.same_bits(b3, w_b)
        avg4, mx4, none = s.error(hto, want_residuals=False)
        assert none is None and gu.same_bits(np.float64(avg4), np.float64(w_avg)) and mx4 == w_max
    finally:
        s.close()
    if per_pair >= 9000:
        assert 2 * len(pts) > 600000             # rows of J


def test_ba_step_lm_sequence(engine, orc):
    """error(state) -> normal_equations -> error(rejected state) -> normal_equations: the second b is J at the
    state times the REJECTED state's residuals (optimize() keeps err_stat from the rejected calcError, :146-153)."""
    n_cam, per_pair, seed, extra = 8, 300, 2, 6
    cams, pairs, pts = ba_case(n_cam, per_pair, seed, extra_pairs=extra)
    mats = numpy_pair_mats(cams, pairs)
    hto2 = numpy_pair_mats(bs.rejected_cams(cams, 5), pairs)[:, 0]
    w1 = _want(orc, n_cam, pairs, mats, mats[:, 0], pts)
    w2 = _want(orc, n_cam, pairs, mats, hto2, pts)
    assert not gu.same_bits(w1[5], w2[5])
    s = engine.ba_session(n_cam, pairs, pts)
    try:
        for hto, (w_res, w_avg, w_max, _, w_jtj, w_b) in ((mats[:, 0], w1), (hto2, w2)):
            avg, mx, res = s.error(hto)
            assert gu.same_bits(res, w_res) and avg == w_avg and mx == w_max
            jtj, b, _ = s.normal_equations(mats)
            assert gu.same_bits(jtj, w_jtj) and gu.same_bits(b, w_b)
    finally:
        s.close()


def test_ba_step_zero_matches(engine, orc):
    """Pairs without matches contribute nothing; a session without any match gives avg = 0/0 = NaN (compared
    with isnan: the default NaN of x86 and of the GPU need not share a sign bit), max 0, J^T J and b zero."""
    cams, pairs, pts = ba_case(4, 30, 9, extra_pairs=2)
    mats = numpy_pair_mats(cams, pairs)
    cut = pairs[0][2]
    pairs2 = [pairs[0], (pairs[1][0], pairs[1][1], 0)] + pairs[2:-1] + [(pairs[-1][0], pairs[-1][1], 0)]
    pts2 = np.concatenate([pts[:cut], pts[cut + pairs[1][2]:len(pts) - pairs[-1][2]]], 0)
    w_res, w_avg, w_max, w_rows, w_jtj, w_b = _want(orc, 4, pairs2, mats, mats[:, 0], pts2)
    s = engine.ba_session(4, pairs2, pts2)
    try:
        avg, mx, res = s.error(mats[:, 0])
        assert gu.same_bits(res, w_res) and avg == w_avg and mx == w_max
        jtj, b, rows = s.normal_equations(mats, want_rows=True)
        assert gu.same_bits(rows, w_rows) and gu.same_bits(jtj, w_jtj) and gu.same_bits(b, w_b)
    finally:
        s.close()
    empty = [(0, 1, 0), (2, 1, 0)]
    s = engine.ba_session(3, empty, np.zeros((0, 4)))
    try:
        avg, mx, res = s.error(np.tile(np.eye(3).reshape(1, 9), (2, 1)))
        w_res, w_avg, w_max = bs.orc_error(empty, np.tile(np.eye(3).reshape(1, 9), (2, 1)), np.zeros((0, 4)))
        assert len(res) == 0 and np.isnan(avg) and np.isnan(w_avg) and mx == w_max == 0.0
        jtj, b, _ = s.normal_equations(np.zeros((2, 13, 9)))
        assert jtj.shape == (18, 18) and not jtj.any() and gu.same_bits(b, np.zeros(18))
    finally:
        s.close()


def test_ba_step_z_zero(engine, orc):
    """A pair whose Hto_to_from gives z = 0: its residuals are infinite.  Every column of b of the other cameras
    is NaN (0 * inf in the reference's dense product); the columns of the pair's two cameras are the sums
    the reference forms (+-inf or NaN).  Residuals, avg, max, J and J^T J stay bit-exact."""
    cams, pairs, pts = ba_case(5, 60, 13, extra_pairs=2)
    mats = numpy_pair_mats(cams, pairs)
    hto = mats[:, 0].copy()
    hto[2, 6:] = 0.0
    w_res, w_avg, w_max, w_rows, w_jtj, w_b = _want(orc, 5, pairs, mats, hto, pts)
    f, t, _ = pairs[2]
    others = np.array([c not in (f, t) for c in range(5) for _ in range(6)])
    assert not np.isfinite(w_res).all() and np.isnan(w_b[others]).all() and not np.isfinite(w_b).any()
    s = engine.ba_session(5, pairs, pts)
    try:
        avg, mx, res = s.error(hto)
        assert gu.same_bits(res, w_res)
        assert gu.same_bits(np.float64(avg), np.float64(w_avg)) and gu.same_bits(np.float64(mx), np.float64(w_max))
        jtj, b, rows = s.normal_equations(mats, want_rows=True)
        assert gu.same_bits(rows, w_rows) and gu.same_bits(jtj, w_jtj) and same_b(b, w_b)
        avg, mx, res = s.error(mats[:, 0])     # a finite state again: b is finite again
        _, b, _ = s.normal_equations(mats)
        assert np.isfinite(b).all() and gu.same_bits(b, _want(orc, 5, pairs, mats, mats[:, 0], pts)[5])
    finally:
        s.close()


def test_ba_step_invalid_calls(engine):
    from openpano_b200.capi import LIB, PanoError
    cams, pairs, pts = ba_case(4, 20, 3)
    mats = numpy_pair_mats(cams, pairs)
    with pytest.raises(PanoError):
        engine.ba_session(4, [(0, 7, pairs[0][2])] + pairs[1:], pts)              # slot out of range
    with pytest.raises(PanoError):
        engine.ba_session(4, [(1, 1, pairs[0][2])] + pairs[1:], pts)              # from == to
    with pytest.raises(PanoError):
        engine.ba_session(4, pairs, pts[:-1])                                     # coordinates for fewer matches
    s = engine.ba_session(4, pairs, pts)
    try:
        with pytest.raises(PanoError):
            s.normal_equations(mats)                                              # no pano_ba_error yet
        with pytest.raises(PanoError):
            s.error(mats[:-1, 0])                                                 # one matrix short
        s.error(mats[:, 0])
        with pytest.raises(PanoError):
            s.normal_equations(mats[:-1])
        # the C ABI itself refuses a pair count that is not the session's
        d = C.c_double()
        h = np.ascontiguousarray(mats[:, 0]).reshape(-1)
        assert LIB.pano_ba_error(s._h, len(pairs) - 1, h.ctypes.data_as(C.POINTER(C.c_double)), C.byref(d),
                                 C.byref(d), None) == -2
        m = np.ascontiguousarray(mats).reshape(-1)
        out = np.zeros(24 * 24 + 24)
        dp = C.POINTER(C.c_double)
        assert LIB.pano_ba_normal_equations(s._h, len(pairs) + 1, m.ctypes.data_as(dp), out.ctypes.data_as(dp),
                                            out[576:].ctypes.data_as(dp), None) == -2
        s.normal_equations(mats)                                                  # still usable
    finally:
        s.close()
    # a match range that does not follow the previous pair's, through the C ABI
    from openpano_b200._abi import PanoBaLink
    links = (PanoBaLink * 2)()
    links[0].from_, links[0].to, links[0].match_begin, links[0].n_match = 0, 1, 0, 3
    links[1].from_, links[1].to, links[1].match_begin, links[1].n_match = 1, 2, 4, 3
    h = C.c_void_p()
    p6 = np.zeros((6, 4))
    assert LIB.pano_ba_session_create(engine._h, 3, 2, links, p6.ctypes.data_as(C.POINTER(C.c_double)), C.byref(h)) == -2
    assert not h.value


def test_cpp_ba_step_equals_reference_members(tmp_path):
    """B200BundleAdjusterStep (openpano_b200/host/pano_host.hh) next to IncrementalBundleAdjuster's own calcError /
    calcJacobianSymbolic / J^T * err_vec, compiled against the reference's headers (oracle/_ref/ba_step_test)."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/ba_step_test not built (needs the reference sources at build time)")
    cams, pairs, pts = ba_case(6, 150, 21, extra_pairs=4)
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<2i", len(cams), len(pairs)))
        for p in pairs:
            f.write(struct.pack("<3i", *p))
        f.write(np.ascontiguousarray(cams, np.float64).tobytes())
        f.write(np.ascontiguousarray(bs.rejected_cams(cams, 3), np.float64).tobytes())
        f.write(np.ascontiguousarray(pts, np.float64).tobytes())
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(path)], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "BA STEP TEST OK" in out.stdout
    assert "after a rejected step" in out.stdout
