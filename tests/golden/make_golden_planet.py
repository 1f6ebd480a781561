#!/usr/bin/env python
"""Generates tests/golden/planet.npz from the REFERENCE's own planet() (main.cc:294-331, compiled in place
into oracle/_ref/libopenpano_ref_planet.so by oracle/planet.mk with -O2 -ffp-contract=off -msse3).
Per case of tests/planet_util.CASES:

  <name>_case       int32 [w, h, seed]
  <name>_input_sha  SHA-256 of the float32 input (tests/planet_util.make_input)
  <name>_sha        SHA-256 of the reference's float32 1000×1000×3 output
  <name>_sample     the output at the fixed pixels `sample_pos` (N×3 float32), to locate a difference

Run where the reference tree was available at build time (oracle/_ref built):
    python tests/golden/make_golden_planet.py
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))

from tests import golden_util as gu  # noqa: E402
from tests import planet_util as pu  # noqa: E402

OUT = Path(__file__).resolve().parent


def main():
    pos = pu.sample_positions()
    out = {"sample_pos": pos}
    for name, (w, h, seed, holes) in pu.CASES.items():
        img = pu.make_input(w, h, seed, holes)
        res = pu.ref_planet(img)
        out[name + "_case"] = np.array([w, h, seed], np.int32)
        out[name + "_input_sha"] = np.array(gu.sha(img))
        out[name + "_sha"] = np.array(gu.sha(res))
        out[name + "_sample"] = res[pos[:, 0], pos[:, 1]]
        print(f"{name}: {int((res[..., 0] >= 0).sum())} pixels with colour")
    np.savez_compressed(OUT / pu.FIXTURE, **out)
    print(pu.FIXTURE, (OUT / pu.FIXTURE).stat().st_size, "bytes")


if __name__ == "__main__":
    main()
