"""GPU: the little-planet view (pano_planet / pano_planet_dev, main.cc:294-331) against the plain-C restatement
(orc_planet, pinned to the reference's own planet() by tests/test_oracle_planet.py) and against the reference's
digests in tests/golden/planet.npz: all 3·10⁶ floats, raw bits.  Also the device chains it is meant for
(blend -> planet, 8-bit in -> planet -> 8-bit out), the per-context table, invalid calls and the C++ adaptor."""
import ctypes as C
import os
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests import golden_util as gu
from tests import planet_util as pu

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
BIN = ROOT / "oracle" / "_ref" / "planet_test"
OUT_BYTES = pu.SIZE * pu.SIZE * 12


@pytest.mark.parametrize("name", list(pu.CASES))
def test_planet_bit_exact(engine, name):
    img = pu.case_input(name)
    got = engine.planet(img)
    assert gu.same_bits(got, pu.orc_planet(img)), f"{name}: differs from the restatement"
    assert str(gu.load(pu.FIXTURE)[name + "_sha"]) == gu.sha(got), f"{name}: differs from the reference's digest"


def test_planet_dev_equals_host_entry_point(engine):
    """pano_planet_dev on device buffers gives what pano_planet gives; every output float is written (the
    buffer starts as NaN garbage)."""
    img = pu.case_input("holes_1800x300")
    h, w = img.shape[:2]
    d_src, d_out = engine.dev_alloc(img.nbytes), engine.dev_alloc(OUT_BYTES)
    try:
        engine.dev_upload(d_src, img)
        engine.dev_upload(d_out, np.full((pu.SIZE, pu.SIZE, 3), np.nan, np.float32))
        engine.planet_dev(d_src, w, h, d_out)
        got = np.empty((pu.SIZE, pu.SIZE, 3), np.float32)
        engine.dev_download(got, d_out)
    finally:
        engine.dev_free(d_src)
        engine.dev_free(d_out)
    assert gu.same_bits(got, engine.planet(img))
    assert gu.same_bits(got, pu.orc_planet(img))


@pytest.mark.parametrize("bands", [0, 3])
def test_planet_of_blend_dev(engine, orc, bands):
    """pano_blend_dev -> pano_planet_dev without leaving the device equals planet(blend(...)) on the host; the
    serpentine stack leaves uncovered (-1) canvas, so the Color::NO rules apply."""
    imgs, org = synth.make_stack(5, 260, 200, 90, 77, rows=2, step_y=70)
    items, geom = synth.translation_blend_setup(org, 260, 200)
    p = default_params(multiband=bands, lazy_read=0)
    shapes = [im.shape[:2] for im in imgs]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    want_mosaic = orc.blend(imgs, items, geom, bands, p)
    assert (want_mosaic[..., 0] == -1).sum() > 1000
    want = pu.orc_planet(want_mosaic)
    d_imgs = [engine.dev_alloc(im.nbytes) for im in imgs]
    d_mos, d_out = engine.dev_alloc(tw * th * 12), engine.dev_alloc(OUT_BYTES)
    got = np.empty((pu.SIZE, pu.SIZE, 3), np.float32)
    try:
        for d, im in zip(d_imgs, imgs):
            engine.dev_upload(d, im)
        engine.blend_dev(d_imgs, shapes, items, geom, d_mos, tw, th, bands, p)
        engine.planet_dev(d_mos, tw, th, d_out)
        engine.dev_download(got, d_out)
    finally:
        for d in d_imgs + [d_mos, d_out]:
            engine.dev_free(d)
    assert gu.same_bits(got, want)


def test_planet_rgb8_chain(engine, orc):
    """8-bit pixels in -> read_img's conversion -> planet -> write_rgb's conversion of the whole 1000×1000 image,
    all on the device, equals the same three steps of the restatement."""
    pix = (synth.make_canvas(300, 1400, 41) * 255.0 + 0.5).astype(np.uint8)
    h, w = pix.shape[:2]
    want = orc.write_rgb8(pu.orc_planet(orc.read_img_rgb8(pix)))
    d_pix, d_mat = engine.dev_alloc(pix.nbytes), engine.dev_alloc(h * w * 12)
    d_planet, d_rgb8 = engine.dev_alloc(OUT_BYTES), engine.dev_alloc(pu.SIZE * pu.SIZE * 3)
    got = np.empty((pu.SIZE, pu.SIZE, 3), np.uint8)
    try:
        engine.dev_upload(d_pix, pix)
        engine.rgb8_to_mat32f_dev(d_pix, w, h, 3, d_mat)
        engine.planet_dev(d_mat, w, h, d_planet)
        engine.mat32f_to_rgb8_dev(d_planet, pu.SIZE, pu.SIZE, None, d_rgb8)
        engine.dev_download(got, d_rgb8)
    finally:
        for d in (d_pix, d_mat, d_planet, d_rgb8):
            engine.dev_free(d)
    assert np.array_equal(got, want)
    assert (got == 255).all(axis=2).any() and not (got == 255).all()     # Color::NO turned white, the rest not


def test_planet_table_reused_across_calls_and_contexts(engine):
    """The per-pixel table is uploaded once per context: repeated calls on one context, calls with other
    shapes in between and a call on a second context all give the same bits."""
    from openpano_b200.capi import Engine
    img = pu.case_input("tall_600x800")
    other = pu.case_input("w4_1200x400")
    first = engine.planet(img)
    engine.planet(other)
    assert gu.same_bits(engine.planet(img), first)
    eng2 = Engine(0)
    try:
        assert gu.same_bits(eng2.planet(img), first)
        assert gu.same_bits(eng2.planet(img), first)
    finally:
        eng2.close()
    assert gu.same_bits(engine.planet(img), first)        # the first context is unaffected by the second's teardown


def test_planet_invalid_calls(engine):
    from openpano_b200.capi import LIB, PanoError
    fp = C.POINTER(C.c_float)
    img = np.zeros((4, 6, 3), np.float32)
    out = np.empty((pu.SIZE, pu.SIZE, 3), np.float32)
    pi, po = img.ctypes.data_as(fp), out.ctypes.data_as(fp)
    assert LIB.pano_planet(None, pi, 6, 4, po) == -2
    assert LIB.pano_planet(engine._h, None, 6, 4, po) == -2
    assert LIB.pano_planet(engine._h, pi, 6, 4, None) == -2
    assert LIB.pano_planet(engine._h, pi, 0, 4, po) == -2
    assert LIB.pano_planet(engine._h, pi, 6, -1, po) == -2
    d = engine.dev_alloc(OUT_BYTES)
    try:
        assert LIB.pano_planet_dev(None, C.c_void_p(d), 6, 4, C.c_void_p(d)) == -2
        assert LIB.pano_planet_dev(engine._h, None, 6, 4, C.c_void_p(d)) == -2
        assert LIB.pano_planet_dev(engine._h, C.c_void_p(d), 6, 4, None) == -2
        assert LIB.pano_planet_dev(engine._h, C.c_void_p(d), 6, 0, C.c_void_p(d)) == -2
    finally:
        engine.dev_free(d)
    with pytest.raises(PanoError):
        engine.planet(np.zeros((4, 6), np.float32))                       # not H×W×3
    assert gu.same_bits(engine.planet(img), pu.orc_planet(img))           # still usable


def test_cpp_planet_equals_reference_planet(tmp_path):
    """b200_planet (openpano_b200/host/pano_host.hh) next to the reference's own planet(), compiled against the
    reference's headers (oracle/_ref/planet_test)."""
    if not BIN.exists():
        pytest.skip("oracle/_ref/planet_test not built (needs the reference sources at build time)")
    paths = []
    for name in ("holes_1800x300", "mosaic_6488x1100", "tiny_2x2", "column_1x5"):
        img = pu.case_input(name)
        path = tmp_path / f"{name}.bin"
        with open(path, "wb") as f:
            f.write(struct.pack("<2i", img.shape[1], img.shape[0]))
            f.write(img.tobytes())
        paths.append(str(path))
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = f"{ROOT / 'oracle' / '_ref'}:{ROOT / 'openpano_b200'}:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([str(BIN)] + paths, capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "PLANET TEST OK" in out.stdout
    assert out.stdout.count("identical") == len(paths)
