#!/usr/bin/env python
"""Generates the bundle-adjustment LM-iteration fixtures from the REFERENCE's own translation unit
(oracle/_ref/libopenpano_ref_ba_step.so, built by oracle/ba_step.mk from the reference's
stitch/incremental_bundle_adjuster.cc with -O2 -ffp-contract=off -msse3):

  tests/golden/ba_step_5cams.npz   calcError's residuals, avg and max and b = J^T * residuals, at a state and
                                   at a rejected new state (whose residuals the next b uses with the kept
                                   state's J), with the Hto_to_from matrices and the 13 per-pair matrices the
                                   reference's operations made
  tests/golden/ba_step_vs_ref.npz  digests of the same outputs for the cases of tests/test_oracle_ba_step.py

Run where the reference tree was available at build time (oracle/_ref built):
    python tests/golden/make_golden_ba_step.py
"""
import hashlib
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))

from tests import ba_step_util as bs  # noqa: E402
from tests import test_oracle_ba_step as t  # noqa: E402
from tests.ba_util import ba_case  # noqa: E402
from tests.checker import get_checker  # noqa: E402

OUT = Path(__file__).resolve().parent


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def main():
    ref = get_checker("ref")                     # ref_ba_pair_mats: the 13 per-pair matrices
    assert ref.num_threads() == 1
    cams, pairs, pts = ba_case(5, 40, 5, extra_pairs=3)
    cams2 = bs.rejected_cams(cams, 11)
    res, avg, mx, hto = bs.ref_error(cams, pairs, pts)
    res2, avg2, mx2, hto2 = bs.ref_error(cams2, pairs, pts)
    np.savez_compressed(OUT / "ba_step_5cams.npz", input_sha=np.array(sha(cams, np.array(pairs), pts)),
                        mats=ref.ba_pair_mats(cams, pairs), hto=hto, residuals=res, avg=np.float64(avg), max=np.float64(mx),
                        b=bs.ref_jtr(cams, pairs, pts, res), hto_rejected=hto2, residuals_rejected=res2,
                        avg_rejected=np.float64(avg2), max_rejected=np.float64(mx2),
                        b_rejected=bs.ref_jtr(cams, pairs, pts, res2))
    print("ba_step:", len(pairs), "pairs, avg", avg, "rejected avg", avg2)
    out = {}
    for args in t.BA_STEP_CASES:
        cams, pairs, pts = ba_case(*args[:3], extra_pairs=args[3])
        states = [cams, bs.rejected_cams(cams, args[2] + 100)]
        errs = [bs.ref_error(c, pairs, pts) for c in states]
        for tag, (res, avg, mx, hto) in zip(t.STATES, errs):
            out[t.hto_key(tag, *args)] = hto
            out[t.case_key("test_ba_error", tag, *args)] = np.array(t.digests([res, np.array([avg, mx])]))
        out[t.case_key("test_ba_jtr", *args)] = np.array(t.digests([bs.ref_jtr(cams, pairs, pts, e[0]) for e in errs]))
    np.savez_compressed(OUT / t.FIXTURE, **out)
    print("ba_step_vs_ref:", len(out), "entries")


if __name__ == "__main__":
    main()
