"""CPU: the plain-C restatement of the little-planet view, orc_planet (main.cc:294-331), against the reference's
own planet() (ref_planet, oracle/refshim/ref_planet.cc: main.cc compiled in place with its file I/O handed over
in memory) and against tests/golden/planet.npz, which tests/golden/make_golden_planet.py made from that
function: SHA-256 of every input and output, plus a fixed sample of output pixels.  Bit for bit."""
import numpy as np
import pytest

from tests import golden_util as gu
from tests import planet_util as pu

NAMES = list(pu.CASES)


@pytest.mark.parametrize("name", NAMES)
def test_planet_matches_golden(name):
    g = gu.load(pu.FIXTURE)
    w, h, seed, holes = pu.CASES[name]
    assert tuple(g[name + "_case"]) == (w, h, seed)
    img = pu.make_input(w, h, seed, holes)
    assert str(g[name + "_input_sha"]) == gu.sha(img)
    out = pu.orc_planet(img)
    pos = g["sample_pos"]
    assert gu.same_bits(out[pos[:, 0], pos[:, 1]], g[name + "_sample"]), f"{name}: sampled pixels differ"
    assert str(g[name + "_sha"]) == gu.sha(out), f"{name}: output differs from the reference's"


@pytest.mark.parametrize("name", NAMES)
def test_planet_equals_reference(name):
    if not pu.have_ref():
        pytest.skip("oracle/_ref/libopenpano_ref_planet.so not built (needs the reference sources)")
    img = pu.case_input(name)
    assert gu.same_bits(pu.orc_planet(img), pu.ref_planet(img))


def test_planet_shape_rules():
    """The disc: no colour at the centre pixel or at distance >= 500; h == 1 or w == 1 gives no colour at all;
    a hole-free input colours every other pixel of the disc except where the row reaches h - 1 (fr + 1 >= h)
    or the column reaches w - 1 (fc + 1 >= w)."""
    img = pu.case_input("tall_600x800")
    out = pu.orc_planet(img)
    assert (out[500, 500] == -1).all() and (out[0, 0] == -1).all() and (out[500, 0] == -1).all()
    i, j = np.mgrid[0:pu.SIZE, 0:pu.SIZE]
    outside = np.hypot(500 - i, 500 - j) >= 500
    assert (out[outside] == -1).all()
    coloured = out[..., 0] >= 0
    assert coloured.sum() > 0.9 * (~outside).sum()
    assert ((out[coloured] >= 0) & (out[coloured] <= 1)).all()
    for name in ("row_5x1", "column_1x5"):
        assert (pu.orc_planet(pu.case_input(name)) == -1).all(), name
    assert (pu.orc_planet(pu.case_input("tiny_2x2"))[..., 0] >= 0).any()


def test_planet_negative_green_is_not_a_hole():
    """interpolate() tests only the first channel of a tap for Color::NO: a negative green value is mixed in."""
    out = pu.orc_planet(pu.case_input("holes_1800x300"))
    col = out[out[..., 0] >= 0]
    assert (col[:, 1] < 0).any()
