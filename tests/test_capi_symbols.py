"""CPU: the C-ABI library builds, loads, and exports every symbol that
include/pano_b200.h declares; without a GPU the engine fails loudly instead of
falling back to any CPU path."""
import ctypes
import re
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "pano_b200.h"
LIB = ROOT / "openpano_b200" / "libpano_b200.so"


def declared_functions():
    text = HEADER.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(pano_[a-z0-9_]+)\s*\(", text)))


def test_library_is_built():
    assert LIB.exists(), "run python -c 'import __graft_entry__ as g; g.build()'"


def test_every_declared_symbol_is_exported():
    names = declared_functions()
    assert len(names) >= 40
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB)], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (pano_[a-z0-9_]+)", out))
    missing = [n for n in names if n not in exported]
    assert not missing, f"declared in pano_b200.h but not exported: {missing}"
    lib = ctypes.CDLL(str(LIB))
    for n in names:
        getattr(lib, n)


def test_binding_covers_the_header():
    from openpano_b200 import capi
    assert set(declared_functions()) == set(capi.EXPORTED)


def test_library_is_sm90a_with_tensor_core_and_bulk_copy_code():
    out = subprocess.run(["cuobjdump", "-lelf", str(LIB)], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump not available")
    assert "sm_90a" in out.stdout
    sass = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True).stdout
    assert "HGMMA" in sass            # wgmma.mma_async
    assert "UBLKCP" in sass           # cp.async.bulk
    assert "UTMALDG" in sass          # cp.async.bulk.tensor (TMA tile loads)


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    from openpano_b200.capi import Engine, PanoError
    with pytest.raises(PanoError) as ei:
        Engine(0)
    assert ei.value.code == -4        # PANO_ERR_NO_DEVICE


def test_params_default_matches_config_cfg():
    from openpano_b200.capi import LIB as L
    from openpano_b200._abi import PanoParams, default_params
    p = PanoParams()
    L.pano_params_default(ctypes.byref(p))
    q = default_params()
    for name, _ in PanoParams._fields_:
        assert getattr(p, name) == getattr(q, name), name
    assert p.num_octave == 4 and p.num_scale == 7 and p.sift_working_size == 800


def test_host_only_entry_points_work_without_gpu(orc):
    """pano_cyl_warp_shape and pano_blend_target_size are pure host arithmetic."""
    from openpano_b200.capi import Engine
    assert Engine.cyl_warp_shape(600, 400) == orc.cyl_warp_shape(600, 400) == (557, 399, 279.1737406705957, 200.0)
    assert Engine.cyl_warp_shape(257, 311, 1.2) == orc.cyl_warp_shape(257, 311, 1.2)
