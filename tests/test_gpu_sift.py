"""GPU parity of the SIFT chain, stage by stage, against the oracle (plain-C
restatement, pinned to the reference's own TUs in test_oracle_vs_ref.py).
Bit-exact: integer indices AND float planes/descriptors (the engine mirrors the
reference's operation order; see DESIGN.md §3).  Calls go through the C ABI."""
import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests.test_oracle_vs_ref import SIFT_PARAM_SETS, min_points, sift_set_input

pytestmark = pytest.mark.gpu


def _bits(a):
    return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint64) if a.dtype == np.float64 else a


def assert_same(name, a, b):
    assert a.shape == b.shape, (name, a.shape, b.shape)
    if not np.array_equal(_bits(a), _bits(b)):
        diff = np.abs(a.astype(np.float64) - b.astype(np.float64))
        raise AssertionError(f"{name}: {int((a != b).sum())} of {a.size} differ, max abs {diff.max():.3g}")


def compare_trace(g, o, nscale=7, noct=4):
    assert g.working_size() == o.working_size()
    assert_same("working", g.plane(0), o.plane(0))
    for oc in range(noct):
        assert g.octave_size(oc) == o.octave_size(oc)
        for l in range(nscale):
            assert_same(f"gauss[{oc}][{l}]", g.plane(1, oc, l), o.plane(1, oc, l))
        for l in range(nscale - 1):
            assert_same(f"dog[{oc}][{l}]", g.plane(2, oc, l), o.plane(2, oc, l))
    for stage, fields in ((0, ("x", "y", "pyr_id", "scale_id")),
                          (1, ("x", "y", "pyr_id", "scale_id", "real_x", "real_y", "scale_factor")),
                          (2, ("x", "y", "pyr_id", "scale_id", "real_x", "real_y", "scale_factor", "dir"))):
        pg, po = g.points(stage), o.points(stage)
        assert len(pg) == len(po), f"stage {stage}: {len(pg)} vs {len(po)} points"
        for f in fields:
            assert_same(f"stage{stage}.{f}", np.ascontiguousarray(pg[f]), np.ascontiguousarray(po[f]))
    cg, dg = g.descriptors()
    co, do = o.descriptors()
    assert_same("coor", cg, co)
    assert_same("desc", dg, do)
    return len(dg)


@pytest.mark.parametrize("w,h,seed", [(600, 400, 1), (400, 300, 11), (333, 517, 12)])
def test_sift_stages_bit_exact(engine, orc, w, h, seed):
    img = synth.make_canvas(h, w, seed)
    g = engine.sift_trace(img)
    o = orc.sift_trace(img)
    n = compare_trace(g, o)
    assert n > 50
    g.close(); o.close()


def test_sift_baseline_shape_1500x1112(engine, orc):
    imgs, _ = synth.config_stack("ordered_13x1500x1112", n=1)
    g = engine.sift_trace(imgs[0])
    o = orc.sift_trace(imgs[0])
    n = compare_trace(g, o)
    assert n > 500
    g.close(); o.close()


def test_sift_batch_equals_single(engine, orc):
    imgs, _ = synth.make_stack(5, 480, 360, 160, 21)
    imgs.append(synth.make_canvas(300, 420, 22))  # ragged batch: mixed shapes
    fs = engine.sift_detect_batch(imgs)
    for i, im in enumerate(imgs):
        c, d = fs.download(i)
        co, do = orc.sift_detect(im)
        assert_same(f"coor[{i}]", c, co)
        assert_same(f"desc[{i}]", d, do)
    fs.free()


def test_sift_other_params(engine, orc):
    img = synth.make_canvas(360, 480, 31)
    p = default_params(num_octave=3, num_scale=6, contrast_thres=3e-2, edge_ratio=10.0, sift_working_size=500)
    g = engine.sift_trace(img, p)
    o = orc.sift_trace(img, p)
    compare_trace(g, o, nscale=6, noct=3)
    g.close(); o.close()


@pytest.mark.parametrize("hist_scale,ori_radius", [(8, 4.5), (17, 9.0), (20, 4.5)])
def test_sift_wide_descriptor_windows(engine, orc, hist_scale, ori_radius):
    """Descriptor windows wider than one interval-table block of k_descriptor (96 columns: DESC_HIST_SCALE_FACTOR 8
    gives windows of up to ~110 columns, 17 of up to ~215, 20 of up to ~250, close to the 255 the kernel's tables
    hold) and wide orientation windows."""
    img = synth.make_canvas(360, 480, 41)
    p = default_params(desc_hist_scale_factor=hist_scale, ori_radius=ori_radius)
    c, d = engine.sift_detect(img, p)
    co, do = orc.sift_detect(img, p)
    assert len(do) > 300
    assert_same("coor", c, co)
    assert_same("desc", d, do)


def test_sift_flat_image_has_no_features(engine, orc):
    img = np.full((200, 300, 3), 0.5, np.float32)
    c, d = engine.sift_detect(img)
    assert len(d) == 0 and len(orc.sift_detect(img)[1]) == 0


def test_descriptor_properties_full_size(engine):
    """Size-independent properties at a BASELINE shape: RootSIFT rows have L2
    norm 512, entries in [0,512], coordinates inside the image."""
    imgs, _ = synth.config_stack("unordered_38x1300x867", n=2)
    fs = engine.sift_detect_batch(imgs)
    for i in range(2):
        c, d = fs.download(i)
        assert len(d) > 500
        nrm = np.linalg.norm(d.astype(np.float64), axis=1)
        assert np.all(np.abs(nrm - 512.0) < 1e-2)
        assert d.min() >= 0 and d.max() <= 512
        assert np.all(np.abs(c[:, 0]) <= 1300 / 2) and np.all(np.abs(c[:, 1]) <= 867 / 2)
    fs.free()


def test_sift_refuses_windows_beyond_the_tables():
    """The descriptor-radius bound follows OFFSET_THRES: at 6 a refined scale index can pass nscale - 1, and
    DESC_HIST_SCALE_FACTOR 17 (accepted at the default 0.5) gives windows past radius 127."""
    from openpano_b200.capi import Engine, PanoError
    e = Engine(0)
    try:
        with pytest.raises(PanoError) as ei:
            e.sift_detect(synth.make_canvas(180, 260, 31), default_params(desc_hist_scale_factor=17, offset_thres=6.0))
        assert ei.value.code == -2
    finally:
        e.close()


@pytest.mark.parametrize("field,value", SIFT_PARAM_SETS)
def test_sift_param_sets_bit_exact(engine, orc, field, value):
    """The config values tests/test_oracle_vs_ref.py pins to the reference, on the same inputs.  Sets that
    change the planes (NUM_SCALE, GAUSS_SIGMA) are compared stage by stage, the others through the batch
    entry point."""
    img, p = sift_set_input(field, value)
    min_cand, min_desc = min_points(field, value)
    if field in ("num_scale", "gauss_sigma", "all"):
        g, o = engine.sift_trace(img, p), orc.sift_trace(img, p)
        n = compare_trace(g, o, nscale=p.num_scale, noct=p.num_octave)
        assert len(o.points(0)) >= min_cand
        g.close(); o.close()
    else:
        fs = engine.sift_detect_batch([img], p)
        c, d = fs.download(0)
        fs.free()
        co, do = orc.sift_detect(img, p)
        assert_same("coor", c, co)
        assert_same("desc", d, do)
        n = len(d)
    assert n >= min_desc
