"""CPU: the plain-C restatement of one LM iteration's per-point work — orc_ba_error (calcError +
ErrorStats::update_stats, incremental_bundle_adjuster.cc:171-220) and orc_ba_jtr (b = J^T * err_vec,
:237-238) — against the reference's own TU (ref_ba_error / ref_ba_jtr, oracle/refshim/ref_ba_step.cc).
tests/golden/make_golden_ba_step.py ran every case on the reference and stored SHA-256 digests of what it returned in
tests/golden/ba_step_vs_ref.npz, with the Hto_to_from matrices its own operations made (the restatement's
inputs); each test runs the same case on the restatement and compares digests, i.e. bit for bit.  Every case
is checked at a state and at a rejected new state: b always takes J at the state, and the residuals of the
state evaluated last (:140, :152-153)."""
import numpy as np
import pytest

from tests import ba_step_util as bs
from tests import golden_util as gu
from tests.ba_util import ba_case
from tests.test_oracle_vs_ref import BA_CASES, FIXTURE as JACOBIAN_FIXTURE, ba_mats_key, case_key, digests

FIXTURE = "ba_step_vs_ref.npz"
BA_STEP_CASES = BA_CASES          # the Jacobian cases of tests/test_oracle_vs_ref.py: their J is pinned there
STATES = ("state", "rejected")


def hto_key(tag, *params):
    return case_key("ba_hto_" + tag, *params)


def check(key, arrays):
    want = [str(x) for x in gu.load(FIXTURE)[key]]
    got = digests(arrays)
    assert len(got) == len(want), (key, len(got), len(want))
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"{key}: outputs {bad} differ from the reference's"


@pytest.mark.parametrize("n_cam,per_pair,seed,extra", BA_STEP_CASES)
def test_ba_error(n_cam, per_pair, seed, extra):
    """calcError's residuals (trans2d, then from - transformed), update_stats' avg (the sequential sum of
    FLOAT squares) and max, at the state and at the rejected state."""
    _, pairs, pts = ba_case(n_cam, per_pair, seed, extra_pairs=extra)
    g = gu.load(FIXTURE)
    for tag in STATES:
        res, avg, mx = bs.orc_error(pairs, g[hto_key(tag, n_cam, per_pair, seed, extra)], pts)
        assert np.isfinite(res).all() and avg > 0 and mx > 0
        check(case_key("test_ba_error", tag, n_cam, per_pair, seed, extra), [res, np.array([avg, mx])])


@pytest.mark.parametrize("n_cam,per_pair,seed,extra", BA_STEP_CASES)
def test_ba_jtr(orc, n_cam, per_pair, seed, extra):
    """b = J^T * residuals with J at the state, for the state's residuals and for the rejected state's."""
    _, pairs, pts = ba_case(n_cam, per_pair, seed, extra_pairs=extra)
    g = gu.load(FIXTURE)
    mats = gu.load(JACOBIAN_FIXTURE)[ba_mats_key(n_cam, per_pair, seed, extra)]
    rows, _ = orc.ba_jacobian(n_cam, pairs, mats, pts[:, :2])
    bs_ = []
    for tag in STATES:
        res, _, _ = bs.orc_error(pairs, g[hto_key(tag, n_cam, per_pair, seed, extra)], pts)
        bs_.append(bs.orc_jtr(n_cam, pairs, rows, res))
    assert all(np.isfinite(b).all() and (b != 0).any() for b in bs_)
    check(case_key("test_ba_jtr", n_cam, per_pair, seed, extra), bs_)


def test_ba_step_golden_fixture(orc):
    """The restatement against tests/golden/ba_step_5cams.npz (the reference's own outputs, stored whole)."""
    g = gu.load("ba_step_5cams.npz")
    cams, pairs, pts = ba_case(5, 40, 5, extra_pairs=3)
    assert str(g["input_sha"]) == gu.sha(cams, np.array(pairs), pts)
    rows, _ = orc.ba_jacobian(5, pairs, g["mats"], pts[:, :2])
    for sfx in ("", "_rejected"):
        res, avg, mx = bs.orc_error(pairs, g["hto" + sfx], pts)
        assert gu.same_bits(res, g["residuals" + sfx])
        assert gu.same_bits(np.float64(avg), g["avg" + sfx]) and gu.same_bits(np.float64(mx), g["max" + sfx])
        assert gu.same_bits(bs.orc_jtr(5, pairs, rows, res), g["b" + sfx])


def test_ba_error_degenerate():
    """No matches: avg is 0/0 = NaN and max stays 0 (update_stats from avg = max = 0).  A residual that is not
    finite makes every entry of b of the other cameras NaN (0 * inf)."""
    res, avg, mx = bs.orc_error([(0, 1, 0)], np.eye(3).reshape(1, 9), np.zeros((0, 4)))
    assert len(res) == 0 and np.isnan(avg) and mx == 0.0
    _, pairs, pts = ba_case(4, 20, 9)
    hto = np.tile(np.eye(3).reshape(1, 9), (len(pairs), 1))
    hto[1, 6:] = 0.0                                     # z = 0 for every match of pair 1
    res, avg, mx = bs.orc_error(pairs, hto, pts)
    assert not np.isfinite(res[2 * pairs[0][2]:2 * (pairs[0][2] + pairs[1][2])]).any()
    assert np.isfinite(res[:2 * pairs[0][2]]).all() and mx == np.inf
    rows = np.ones((len(pts), 24))
    b = bs.orc_jtr(4, pairs, rows, res).reshape(4, 6)
    f, t, _ = pairs[1]
    assert all(np.isnan(b[c]).all() for c in range(4) if c not in (f, t)) and not np.isfinite(b).any()
