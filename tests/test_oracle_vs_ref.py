"""CPU: the plain-C oracle against the reference's own translation units on inputs beyond the
other fixtures: other shapes, up-sampling, edge cases.  Every case is one function of a checker;
tests/golden/make_golden.py ran it on the reference's TUs (oracle/_ref) and stored SHA-256 digests of
what the reference returned in tests/golden/oracle_vs_ref.npz, and each test runs the same case on
the restatement and compares digests, i.e. bit for bit.  The bundle-adjustment case also stores the
per-pair matrices the reference evaluated: they are the restatement's inputs."""
import hashlib

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params
from tests import golden_util as gu

FIXTURE = "oracle_vs_ref.npz"


def digests(arrays):
    """One SHA-256 per output array, over its dtype, shape and bytes."""
    out = []
    for a in arrays:
        a = np.ascontiguousarray(a)
        h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
        h.update(a.tobytes())
        out.append(h.hexdigest())
    return out


def case_key(name, *params):
    return name + "[" + "-".join(str(p) for p in params) + "]"


def check(key, arrays):
    want = [str(x) for x in gu.load(FIXTURE)[key]]
    got = digests(arrays)
    assert len(got) == len(want), (key, len(got), len(want))
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"{key}: outputs {bad[:10]} differ from the reference's"


# ----------------------------------------------------------------------------- cases
def _trace_outputs(tr, noct=4, nscale=7):
    out = [np.array(tr.working_size()), tr.plane(0)]
    for o in range(noct):
        out.append(np.array(tr.octave_size(o)))
        out += [tr.plane(1, o, l) for l in range(nscale)]
        out += [tr.plane(2, o, l) for l in range(nscale - 1)]
        for l in range(1, nscale):
            out += [tr.plane(3, o, l), tr.plane(4, o, l)]
    out += [np.frombuffer(tr.points(st).tobytes(), np.uint8) for st in range(3)]
    out += list(tr.descriptors())
    tr.close()
    return out


SIFT_STAGES = [(300, 200, 7), (200, 300, 8), (157, 211, 9)]


def case_sift_every_stage(chk, w, h, seed):
    return _trace_outputs(chk.sift_trace(synth.make_canvas(h, w, seed)))


def case_sift_other_params(chk):
    img = synth.make_canvas(180, 260, 31)
    p = default_params(num_octave=3, num_scale=6, contrast_thres=3e-2, edge_ratio=10.0, sift_working_size=300)
    return _trace_outputs(chk.sift_trace(img, p), noct=3, nscale=6)


# Config values off their defaults, each reaching its own device code; "all" changes them at once.
SIFT_PARAM_SETS = [("gauss_sigma", 1.6), ("gauss_sigma", 2.0), ("num_scale", 4), ("num_scale", 5), ("num_scale", 8),
                   ("num_scale", 9), ("num_octave", 8), ("pre_color_thres", 0.01), ("judge_extrema_diff_thres", 0.0),
                   ("judge_extrema_diff_thres", 0.01), ("offset_thres", 0.3), ("ori_hist_smooth_count", 0),
                   ("ori_hist_smooth_count", 5), ("desc_int_factor", 1), ("desc_int_factor", 100),
                   ("desc_int_factor", 4096), ("all", 0)]
ALL_CHANGED = dict(gauss_sigma=1.6, num_scale=9, num_octave=5, pre_color_thres=0.01, judge_extrema_diff_thres=1e-3,
                   calc_offset_depth=8, offset_thres=0.3, ori_hist_smooth_count=0, desc_int_factor=100)


def sift_set_input(field, value):
    """(image, params) of one set.  NUM_SCALE 4 and 5 leave one and two admissible refined scale indices
    (1 <= s <= nscale - 3): on the canvas the pre-colour and contrast thresholds remove every candidate,
    so these two sets run on a uniform-noise image with both thresholds at 0."""
    if field == "num_scale" and value <= 5:
        img = np.random.RandomState(31).rand(180, 260, 3).astype(np.float32)
        return img, default_params(num_scale=value, pre_color_thres=0.0, contrast_thres=0.0)
    return synth.make_canvas(180, 260, 31), default_params(**(ALL_CHANGED if field == "all" else {field: value}))


def min_points(field, value):
    """(extremum candidates, descriptors) each set keeps at least on its input (the canvas keeps 171
    descriptors at the defaults)."""
    if field == "num_scale" and value <= 5:
        return 100, 30
    if field == "judge_extrema_diff_thres" and value > 2e-3:
        return 1, 1
    return 100, 100


def case_sift_param_set(chk, field, value):
    img, p = sift_set_input(field, value)
    return _trace_outputs(chk.sift_trace(img, p), noct=p.num_octave, nscale=p.num_scale)


WIDE_WINDOWS = [(8, 4.5), (17, 9.0), (20, 4.5)]


def case_sift_wide_windows(chk, hist_scale, ori_radius):
    img = synth.make_canvas(200, 280, 41)
    return list(chk.sift_detect(img, default_params(desc_hist_scale_factor=hist_scale, ori_radius=ori_radius)))


def case_sift_flat_image(chk):
    return list(chk.sift_detect(np.full((120, 160, 3), 0.25, np.float32)))


def case_match_ragged_and_ties(chk):
    rng = np.random.RandomState(3)
    a = synth.rootsift_like(260, 5)
    b = np.concatenate([a[:80], a[:80], a[150:]])                   # exact duplicates: zero-distance ties
    noisy = (a[rng.permutation(260)][:200] + rng.randn(200, 128).astype(np.float32) * 36).astype(np.float32)
    return [chk.match(x, y) for x, y in ((a, b), (b, a), (a, noisy), (noisy, a), (a[:1], b), (b, a[:1]), (a[:2], a[:2]))]


CYL_WARPS = [(200, 140, 1.0), (141, 173, 0.8), (160, 120, 1.3)]


def case_cyl_warp(chk, w, h, hf):
    img = synth.make_canvas(h, w, 61)
    k = np.array([[3.5, -2.25], [-60.0, 40.0]])
    return [np.array(chk.cyl_warp_shape(w, h, hf)), *chk.cyl_warp(img, k, hf)]


def case_blend_projections(chk, projection, bands):
    import math
    imgs, org = synth.make_stack(3, 160, 110, 60, 71)
    items = []
    for k, (x, y) in enumerate(org):
        if projection == 0:
            th = 0.003 * (k - 1)
            H = np.array([[math.cos(th), -math.sin(th), x - 80], [math.sin(th), math.cos(th), 2 * k], [1e-5 * k, -2e-5, 1.0]])
        else:
            f = 300.0
            H = np.array([[1 / f, 0, (x - 80) / f], [0, 1 / f, 0.004 * k], [0, 0, 1]])
        items.append((k * 60, 0, k * 60 + 160, 115, list(np.linalg.inv(H).ravel())))
    res = 1.0 if projection == 0 else 1 / 300.0
    pmin = (-80.0, -55.0) if projection == 0 else (-0.3, -0.2)
    geom = dict(projection=projection, res_x=res, res_y=res, proj_min_x=pmin[0], proj_min_y=pmin[1])
    return [chk.blend(imgs, items, geom, bands)]


def _random_mosaic(rng, h, w):
    m = rng.rand(h, w, 3).astype(np.float32)
    for _ in range(rng.randint(0, 6)):
        y0, x0 = rng.randint(0, h), rng.randint(0, w)
        m[y0:y0 + rng.randint(1, 8), x0:x0 + rng.randint(1, 10)] = -1
    if rng.rand() < 0.4:
        m[:rng.randint(0, 4)] = -1
        m[:, :rng.randint(0, 5)] = -1
    return m


def case_imgio_read_write(chk):
    """read_img / write_rgb (the reference's imgio.cc through lossless PNM files)."""
    rng = np.random.RandomState(11)
    allv = np.arange(256, dtype=np.uint8).reshape(16, 16)
    out = [chk.read_img_rgb8(pix) for pix in (rng.randint(0, 256, (37, 53, 3)).astype(np.uint8), np.stack([allv] * 3, -1),
                                               allv, rng.randint(0, 256, (9, 31)).astype(np.uint8))]
    m = _random_mosaic(rng, 40, 60)
    m[0, 0] = (1.0, 0.0, 0.999999)
    m[0, 1] = np.float32(1.0) / np.float32(255.0) * np.arange(1, 4, dtype=np.float32)
    return out + [chk.write_rgb8(m)]


def crop_cases():
    rng = np.random.RandomState(12)
    cases = [_random_mosaic(rng, rng.randint(5, 60), rng.randint(5, 90)) for _ in range(25)]
    cases.append(-np.ones((6, 7, 3), np.float32))                  # nothing valid: 0 x 1 result
    cases.append(rng.rand(8, 9, 3).astype(np.float32))              # everything valid
    return cases


def case_imgio_crop(chk):
    out = []
    for m in crop_cases():
        rect, cropped = chk.crop(m)                                 # x0, y0 are -1 from the reference's build
        out += [rect[2:], cropped]
    return out


MATCH_RATIOS = [(0.6, 1, 60), (0.95, 150, 190), (0.5, 60, 150), (1.0, 189, 190)]
RATIO_NOISE = {0.5: 20.0}        # at noise 30 ratio 0.5 accepts nothing


def case_match_other_ratios(chk, ratio, noise=None):
    noise = RATIO_NOISE.get(ratio, 30.0) if noise is None else noise
    rng = np.random.RandomState(21)
    a = synth.rootsift_like(220, 22)
    b = (a[rng.permutation(220)][:190] + rng.randn(190, 128).astype(np.float32) * np.float32(noise)).astype(np.float32)
    p = default_params(match_reject_next_ratio=ratio)
    return [chk.match(a, b, p), chk.match(b, a, p)]


SCALED_BLENDS = [(0, 0), (1, 1)]


def case_blend_scaled_resolution(chk, lazy, ordered):
    imgs, org = synth.make_stack(3, 200, 150, 80, 73)
    items, geom = synth.translation_blend_setup(org, 200, 150, max_output_size=170)
    assert geom["res_x"] > 2.0
    p = default_params(lazy_read=lazy, ordered_input=ordered)
    return [chk.blend(imgs, items, geom, 0, p), chk.blend(imgs, items, geom, 3, p)]


def case_blend_window_factor(chk, factor):
    """GAUSS_WINDOW_FACTOR in the multiband blender: its taps and the halo of every band."""
    imgs, org = synth.make_stack(3, 160, 110, 60, 71)
    items, geom = synth.translation_blend_setup(org, 160, 110)
    return [chk.blend(imgs, items, geom, 3, default_params(multiband=3, gauss_window_factor=factor))]


def case_cyl_warp_other_focal(chk):
    img = synth.make_canvas(120, 180, 62)
    p = default_params(focal_length=24.0)
    k = np.array([[10.0, 5.0], [-80.0, -50.0]])
    return [np.array(chk.cyl_warp_shape(180, 120, 1.0, p)), *chk.cyl_warp(img, k, 1.0, p)]


RANSAC_CASES = [(300, 200, 1), (8, 50, 2), (1200, 64, 3)]


def case_ransac_scoring(chk, n_match, n_hyp, seed):
    from tests.ransac_util import ransac_case
    best, count, counts, flags = chk.ransac_score(*ransac_case(n_match, n_hyp, seed))
    return [np.array([best, count]), counts, flags]


BA_CASES = [(4, 50, 1, 2), (8, 300, 2, 6), (3, 1, 3, 0), (16, 1000, 4, 30)]


def ba_mats_key(n_cam, per_pair, seed, extra):
    return case_key("ba_pair_mats", n_cam, per_pair, seed, extra)


# (golden key, case function, case arguments) of every stored case: make_golden.py runs these on the
# reference.  The MATCH_RATIOS cases are generated one per process: the reference squares the ratio
# into a function-local `static const` on its first call (matcher.cc:16, :91).
def golden_cases():
    cases = [(case_key("test_sift_every_stage", *a), case_sift_every_stage, a) for a in SIFT_STAGES]
    cases += [("test_sift_other_params", case_sift_other_params, ()),
              ("test_sift_flat_image", case_sift_flat_image, ()),
              ("test_match_ragged_and_ties", case_match_ragged_and_ties, ()),
              ("test_imgio_read_write", case_imgio_read_write, ()),
              ("test_imgio_crop", case_imgio_crop, ()),
              ("test_cyl_warp_other_focal", case_cyl_warp_other_focal, ())]
    cases += [(case_key("test_sift_wide_windows", *a), case_sift_wide_windows, a) for a in WIDE_WINDOWS]
    cases += [(case_key("test_sift_param_set", *a), case_sift_param_set, a) for a in SIFT_PARAM_SETS]
    cases += [(case_key("test_blend_window_factor", f), case_blend_window_factor, (f,)) for f in (4,)]
    cases += [(case_key("test_cyl_warp", *a), case_cyl_warp, a) for a in CYL_WARPS]
    cases += [(case_key("test_blend_projections", p, b), case_blend_projections, (p, b)) for p in (0, 1, 2) for b in (0, 2)]
    cases += [(case_key("test_blend_scaled_resolution", *a), case_blend_scaled_resolution, a) for a in SCALED_BLENDS]
    cases += [(case_key("test_ransac_scoring", *a), case_ransac_scoring, a) for a in RANSAC_CASES]
    return cases


# ----------------------------------------------------------------------------- tests
@pytest.mark.parametrize("w,h,seed", SIFT_STAGES)
def test_sift_every_stage(orc, w, h, seed):
    out = case_sift_every_stage(orc, w, h, seed)
    assert len(out[-1]) > 20
    check(case_key("test_sift_every_stage", w, h, seed), out)


def test_sift_other_params(orc):
    check("test_sift_other_params", case_sift_other_params(orc))


@pytest.mark.parametrize("field,value", SIFT_PARAM_SETS)
def test_sift_param_set(orc, field, value):
    """Every stage at one config value off its default; the result must differ from the defaults' on the
    same image, or the case would pin nothing.  (CALC_OFFSET_DEPTH alone leaves these images' features
    unchanged: it is part of the "all" set.)"""
    out = case_sift_param_set(orc, field, value)
    img, p = sift_set_input(field, value)
    base = _trace_outputs(orc.sift_trace(img))
    assert not (np.array_equal(out[-2], base[-2]) and np.array_equal(out[-1], base[-1]))
    tr = orc.sift_trace(img, p)
    n_cand = len(tr.points(0))
    tr.close()
    min_cand, min_desc = min_points(field, value)
    assert n_cand >= min_cand and len(out[-1]) >= min_desc, (n_cand, len(out[-1]))
    check(case_key("test_sift_param_set", field, value), out)


@pytest.mark.parametrize("hist_scale,ori_radius", WIDE_WINDOWS)
def test_sift_wide_windows(orc, hist_scale, ori_radius):
    """The parameter sets tests/test_gpu_sift.py::test_sift_wide_descriptor_windows runs on the GPU (descriptor
    windows wider than one interval-table block of the kernel, wide orientation windows): the restatement
    against the reference's own TUs, so that the GPU-vs-oracle result there is pinned to the reference too."""
    out = case_sift_wide_windows(orc, hist_scale, ori_radius)
    assert len(out[1]) > 100
    check(case_key("test_sift_wide_windows", hist_scale, ori_radius), out)


def test_sift_flat_image(orc):
    out = case_sift_flat_image(orc)
    assert len(out[1]) == 0
    check("test_sift_flat_image", out)


def test_match_ragged_and_ties(orc):
    check("test_match_ragged_and_ties", case_match_ragged_and_ties(orc))


@pytest.mark.parametrize("w,h,hf", CYL_WARPS)
def test_cyl_warp(orc, w, h, hf):
    check(case_key("test_cyl_warp", w, h, hf), case_cyl_warp(orc, w, h, hf))


@pytest.mark.parametrize("projection", [0, 1, 2])
@pytest.mark.parametrize("bands", [0, 2])
def test_blend_projections(orc, projection, bands):
    out = case_blend_projections(orc, projection, bands)
    assert (out[0] >= 0).mean() > 0.3
    check(case_key("test_blend_projections", projection, bands), out)


def test_imgio_read_write(orc):
    check("test_imgio_read_write", case_imgio_read_write(orc))


def test_imgio_crop(orc):
    for m in crop_cases():
        (x0, y0, cw, ch), cropped = orc.crop(m)
        assert np.array_equal(cropped, m[y0:y0 + ch, x0:x0 + cw])
    check("test_imgio_crop", case_imgio_crop(orc))


@pytest.mark.parametrize("ratio,lo,hi", MATCH_RATIOS)
def test_match_other_ratios(orc, ratio, lo, hi):
    """MATCH_REJECT_NEXT_RATIO is a config value (config.cfg:33); the restatement takes it per call."""
    out = case_match_other_ratios(orc, ratio)
    assert lo <= len(out[0]) <= hi
    assert not np.array_equal(out[0], case_match_other_ratios(orc, 0.8, RATIO_NOISE.get(ratio, 30.0))[0])
    check(case_key("test_match_other_ratios", ratio), out)


@pytest.mark.parametrize("lazy,ordered", SCALED_BLENDS)
def test_blend_scaled_resolution(orc, lazy, ordered):
    """MAX_OUTPUT_SIZE shrinks the canvas through `resolution` (stitcher_image.cc:108-119): the
    blend map then samples the sources at a stride > 1."""
    out = case_blend_scaled_resolution(orc, lazy, ordered)
    assert (out[0] >= 0).mean() > 0.5
    check(case_key("test_blend_scaled_resolution", lazy, ordered), out)


def test_blend_window_factor(orc):
    out = case_blend_window_factor(orc, 4)
    assert not gu.same_bits(out[0], case_blend_window_factor(orc, 6)[0])
    check(case_key("test_blend_window_factor", 4), out)


def test_cyl_warp_other_focal(orc):
    check("test_cyl_warp_other_focal", case_cyl_warp_other_focal(orc))


def test_oracle_mt_equals_oracle(orc):
    """oracle/liboracle_mt.so (independent loops under OpenMP, used by the BASELINE-size GPU
    parity tests) must be bit-identical to the single-thread restatement."""
    from tests.checker import get_checker, have
    if not have("orc_mt"):
        pytest.skip("oracle/liboracle_mt.so not built")
    mt = get_checker("orc_mt")
    rng = np.random.RandomState(21)
    a = synth.rootsift_like(900, 4)
    b = a[rng.permutation(900)][:700] + rng.randn(700, 128).astype(np.float32) * 25.0
    for x, y in ((a, b), (b, a), (a[:1], b), (a, a)):
        assert np.array_equal(orc.match(x, y), mt.match(x, y))
    imgs, org = synth.make_stack(5, 260, 200, 90, 77, rows=2, step_y=70)
    items, geom = synth.translation_blend_setup(org, 260, 200)
    for bands in (0, 2, 5):
        for lazy in (0, 1):
            p = default_params(lazy_read=lazy, multiband=bands)
            assert gu.same_bits(orc.blend(imgs, items, geom, bands, p), mt.blend(imgs, items, geom, bands, p)), (bands, lazy)


@pytest.mark.parametrize("n_match,n_hyp,seed", RANSAC_CASES)
def test_ransac_scoring(orc, n_match, n_hyp, seed):
    """TransformEstimation::get_inliers (the reference TU, reached through the shim) against the
    restatement: per-hypothesis counts, first-maximum selection, inlier flags."""
    out = case_ransac_scoring(orc, n_match, n_hyp, seed)
    assert out[0][1] > 0.5 * n_match
    check(case_key("test_ransac_scoring", n_match, n_hyp, seed), out)


@pytest.mark.parametrize("n_cam,per_pair,seed,extra", BA_CASES)
def test_ba_jacobian(orc, n_cam, per_pair, seed, extra):
    """IncrementalBundleAdjuster::calcJacobianSymbolic itself (the reference TU, compiled where it lies
    by oracle/refshim/ref_ba.cc) against the restatement: every J row and every J^T J entry, bit for bit —
    including reversed pairs, repeated camera pairs and the identity camera's small-angle branch.  The
    restatement starts from the per-pair matrices the reference's own Homography / Camera operations made."""
    from tests.ba_util import ba_case
    _, pairs, pts = ba_case(n_cam, per_pair, seed, extra_pairs=extra)
    mats = gu.load(FIXTURE)[ba_mats_key(n_cam, per_pair, seed, extra)]
    rows, jtj = orc.ba_jacobian(n_cam, pairs, mats, pts[:, :2])
    assert np.isfinite(rows).all() and (jtj != 0).any()
    check(case_key("test_ba_jacobian", n_cam, per_pair, seed, extra), [rows, jtj])
