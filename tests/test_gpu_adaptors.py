"""GPU: the drop-in's compiled C++ host (openpano_b200/host/pano_host.hh — subclasses of the
reference's FeatureDetector / BlenderBase, PairWiseMatcher- and CylinderWarper-shaped classes,
a Stitcher::build()-shaped chain) against the reference classes they replace, linked into one
program (oracle/_ref/adaptor_test, built by oracle/Makefile from tests/adaptor/adaptor_test.cc
against the reference's headers).  Everything must be bit-identical."""
import os
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "adaptor_test"


def test_cpp_adaptors_equal_reference_classes(tmp_path):
    if not BIN.exists():
        pytest.skip("oracle/_ref/adaptor_test not built (needs the reference sources at build time)")
    imgs, org = synth.make_stack(4, 360, 270, 120, 47)
    items, geom = synth.translation_blend_setup(org, 360, 270)
    path = tmp_path / "stack.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<3i", len(imgs), 360, 270))
        for im in imgs:
            f.write(np.ascontiguousarray(im, np.float32).tobytes())
        for it in items:
            f.write(struct.pack("<4i", *it[:4]))
            f.write(struct.pack("<9d", *it[4]))
        f.write(struct.pack("<3d", geom["res_x"], geom["proj_min_x"], geom["proj_min_y"]))
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN), str(path)], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "ADAPTOR TEST OK" in out.stdout
    assert "B200Stitcher::build" in out.stdout
