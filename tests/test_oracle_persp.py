"""CPU: the plain-C correction pass (oracle/orc_persp.c) equals the reference's own
CylinderStitcher::perspective_correction (cylstitcher.cc:139-180, reached through a test subclass that sets its
bundle, oracle/refshim/ref_persp.cc) bit for bit, under both LAZY_READ branches and both ORDERED_INPUT values, on
mosaics with Color::NO holes and corrections that keep, keystone, flip, negate or cross z."""
import numpy as np
import pytest

from tests import golden_util as gu
from tests import persp_util as pu

CASES = ["near", "random", "keystone", "keystone_down", "flip", "negative_z", "z_cross"]


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("lazy,ordered", [(1, 1), (1, 0), (0, 1), (0, 0)])
def test_oracle_equals_reference(name, lazy, ordered):
    if not pu.have_ref():
        pytest.skip("oracle/_ref/libopenpano_ref_persp.so not built (needs the reference sources)")
    w, h = 157, 93
    mosaic = pu.mosaic_with_holes(w, h, seed=len(name))
    inv = pu.inv_cases(w, h, seed=3)[name]
    want = pu.ref_correct(mosaic, inv, lazy, ordered)
    got = pu.orc_correct(mosaic, inv, lazy, ordered)
    assert gu.same_bits(got, want), (name, lazy, ordered)
    if name in ("near", "keystone"):
        assert (want[..., 0] >= 0).mean() > 0.5            # most of the canvas is colour, not Color::NO


def test_oracle_matches_golden_fixture():
    """The reference's corrected mosaics, kept as a fixture (tests/golden/cyl_persp.npz): the oracle reproduces
    them without the reference sources."""
    g = gu.load("cyl_persp.npz")
    for key in ("mild", "keystone"):
        got = pu.orc_correct(g["mosaic"], g[f"{key}_inv"], int(g["lazy"]), int(g["ordered"]))
        assert gu.same_bits(got, g[f"{key}_want"]), key
