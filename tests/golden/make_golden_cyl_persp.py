#!/usr/bin/env python
"""Generates tests/golden/cyl_persp.npz from the REFERENCE's own translation units: a small cylinder stack (3
views of 80×60, read_img's values of 8-bit pixels) warped by CylinderWarper and blended by LinearBlender
(oracle/_ref/libopenpano_ref.so), then CylinderStitcher::perspective_correction
(oracle/_ref/libopenpano_ref_persp.so, oracle/cyl_sweep.mk) under two corrections:

  pix                3×80×120×3 uint8 sources;  items_box 3×4 int32, items_inv 3×9 float64;  geom_min 2 float64
  mosaic             the reference's f32 mosaic of the stack
  <key>_inv          the correction's inv: "mild" near the identity, "keystone" strongly keystoned, so that a
                     strip of corrected rows reads a band of mosaic rows many times taller
  <key>_want         the reference's corrected f32 mosaic
  lazy, ordered      the LAZY_READ / ORDERED_INPUT values used

Run where the reference tree was available at build time (oracle/_ref built):
    python tests/golden/make_golden_cyl_persp.py
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))

from openpano_b200 import synth  # noqa: E402
from openpano_b200._abi import default_params  # noqa: E402
from tests import persp_util as pu  # noqa: E402
from tests.checker import get_checker  # noqa: E402

OUT = Path(__file__).resolve().parent
LAZY, ORDERED = 1, 0


def stack():
    """(pix, items, geom, mosaic) of the fixture's cylinder stack through the reference."""
    ref = get_checker("ref")
    imgs, org = synth.make_stack(3, 80, 60, 30, 211)
    pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
    params = default_params(lazy_read=LAZY, ordered_input=ORDERED)
    f32 = [ref.read_img_rgb8(x) for x in pix]
    warped = [ref.cyl_warp(im, np.zeros((0, 2)), 1.0, params)[0] for im in f32]
    oh, ow = warped[0].shape[:2]
    items, geom = synth.translation_blend_setup(org, ow, oh)
    return pix, items, geom, ref.blend(warped, items, geom, 0, params)


def main():
    pix, items, geom, mosaic = stack()
    h, w = mosaic.shape[:2]
    out = {"pix": np.stack(pix), "items_box": np.array([it[:4] for it in items], np.int32),
           "items_inv": np.array([it[4] for it in items], np.float64),
           "geom_min": np.array([geom["proj_min_x"], geom["proj_min_y"]], np.float64),
           "mosaic": mosaic, "lazy": np.int32(LAZY), "ordered": np.int32(ORDERED)}
    for key, inv in (("mild", pu.inv_cases(w, h, 5)["random"]), ("keystone", pu.keystone(w, h, 0.6, 0.0, 0.1))):
        out[f"{key}_inv"] = inv
        out[f"{key}_want"] = pu.ref_correct(mosaic, inv, LAZY, ORDERED)
    np.savez_compressed(OUT / "cyl_persp.npz", **out)
    print(f"wrote {OUT / 'cyl_persp.npz'}: mosaic {w}x{h}")


if __name__ == "__main__":
    main()
