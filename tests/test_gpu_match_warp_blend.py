"""GPU parity of matching, cylinder warp and both blenders against the oracle."""
import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200._abi import default_params

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["auto", "columns_on_demand", "both_sides_first"])
def match_mode(request, monkeypatch):
    """The matcher picks by size whether the larger sets' rows go through the first tensor pass or
    are nominated on request (match.cu: PANO_MATCH_LAZY); both ways must give the reference's pairs."""
    if request.param == "auto":
        monkeypatch.delenv("PANO_MATCH_LAZY", raising=False)
    else:
        monkeypatch.setenv("PANO_MATCH_LAZY", "1" if request.param == "columns_on_demand" else "0")
    return request.param


def test_match_pairs_bit_exact(engine, orc, match_mode):
    imgs, _ = synth.make_stack(4, 480, 360, 160, 41)
    fs = engine.sift_detect_batch(imgs)
    descs = [fs.download(i)[1] for i in range(4)]
    pairs = [(0, 1), (1, 0), (1, 2), (2, 3), (0, 3), (3, 1)]
    got = engine.match_pairs(fs, pairs)
    for (i, j), m in zip(pairs, got):
        want = orc.match(descs[i], descs[j])
        assert np.array_equal(m, want), (i, j, len(m), len(want))
    assert sum(len(m) for m in got) > 100
    assert engine.match_pairs_dev(fs, pairs) == sum(len(m) for m in got)
    fs.free()


@pytest.mark.parametrize("n,m,noise", [(700, 600, 6.0), (600, 700, 25.0), (257, 1000, 40.0), (64, 64, 60.0), (1, 5, 1.0), (5, 1, 1.0)])
def test_match_bruteforce_near_threshold(engine, orc, n, m, noise, match_mode):
    rng = np.random.RandomState(n + m)
    a = synth.rootsift_like(max(n, m), 4)
    b = a[rng.permutation(len(a))][:m] + rng.randn(m, 128).astype(np.float32) * noise
    a = a[:n]
    got = engine.match_bruteforce(a, b)
    want = orc.match(a, b)
    assert np.array_equal(got, want), (len(got), len(want))


def test_match_duplicates_and_ties(engine, orc, match_mode):
    a = synth.rootsift_like(300, 5)
    b = np.concatenate([a[:100], a[:100], a[200:]])  # exact duplicates -> zero-distance ties
    assert np.array_equal(engine.match_bruteforce(a, b), orc.match(a, b))
    assert np.array_equal(engine.match_bruteforce(b, a), orc.match(b, a))


@pytest.mark.parametrize("parts", ["2", "3", "8"])
@pytest.mark.parametrize("lazy", ["0", "1"])
def test_match_first_pass_column_ranges(engine, orc, monkeypatch, parts, lazy):
    """PANO_MATCH_PARTS splits every first-pass task into column ranges merged in k_refine (tail
    balance on large runs).  Exact duplicates placed in different ranges tie on the score: the
    lowest column has to win, as in one range."""
    rng = np.random.RandomState(11)
    a = synth.rootsift_like(1100, 12)
    far = synth.rootsift_like(2400, 13)
    b = np.concatenate([a[:150], far[:1200], a[:150], far[1200:], a[100:400] + rng.randn(300, 128).astype(np.float32) * 15.0])
    monkeypatch.setenv("PANO_MATCH_PARTS", parts)
    monkeypatch.setenv("PANO_MATCH_LAZY", lazy)
    got_ab, got_ba = engine.match_bruteforce(a, b), engine.match_bruteforce(b, a)
    monkeypatch.delenv("PANO_MATCH_PARTS", raising=False)
    monkeypatch.delenv("PANO_MATCH_LAZY", raising=False)
    assert np.array_equal(got_ab, orc.match(a, b))
    assert np.array_equal(got_ba, orc.match(b, a))
    assert len(got_ab) > 50


def test_match_row_shards_concatenate(engine, orc):
    """pano_match_pairs_shard: share s of S of every pair's smaller set; the shares' lists in shard
    order are the unsharded lists (the multi-GPU split of FeatureMatcher::match's loop over k)."""
    rng = np.random.RandomState(5)
    a = synth.rootsift_like(900, 9)
    b = a[rng.permutation(900)][:700] + rng.randn(700, 128).astype(np.float32) * 20.0
    c = np.concatenate([a[:300] + rng.randn(300, 128).astype(np.float32) * 8.0, synth.rootsift_like(250, 10)])
    fs = engine.featureset_upload([a, b, c])
    pairs = [(0, 1), (1, 2), (2, 0), (1, 0)]
    full = engine.match_pairs(fs, pairs)
    sets = [a, b, c]
    for (i, j), m in zip(pairs, full):
        assert np.array_equal(m, orc.match(sets[i], sets[j])), (i, j)
    assert sum(len(m) for m in full) > 300
    for S in (2, 3, 7):
        parts = [engine.match_pairs(fs, pairs, shard=(s, S)) for s in range(S)]
        for k in range(len(pairs)):
            assert np.array_equal(np.concatenate([p[k] for p in parts]), full[k]), (S, k)
        assert sum(engine.match_pairs_dev(fs, pairs, shard=(s, S)) for s in range(S)) == sum(len(m) for m in full)
    fs.free()


def test_match_empty(engine, match_mode):
    a = synth.rootsift_like(10, 6)
    assert len(engine.match_bruteforce(a, np.zeros((0, 128), np.float32))) == 0


@pytest.mark.parametrize("w,h,hf,focal", [(600, 400, 1.0, 37.0), (300, 200, 0.85, 37.0), (257, 311, 1.2, 37.0),
                                          (300, 200, 1.0, 24.0), (257, 311, 0.85, 50.0)])
def test_cyl_warp_bit_exact(engine, orc, w, h, hf, focal):
    """FOCAL_LENGTH sets the cylinder radius (warp.cu)."""
    img = synth.make_canvas(h, w, 51)
    k = np.array([[10.5, -20.25], [-100.0, 50.0], [0.0, 0.0]])
    p = default_params(focal_length=focal)
    assert engine.cyl_warp_shape(w, h, hf, p) == orc.cyl_warp_shape(w, h, hf, p)
    ga, gk = engine.cyl_warp(img, k, hf, p)
    oa, ok = orc.cyl_warp(img, k, hf, p)
    assert np.array_equal(gk, ok)
    assert ga.shape == oa.shape
    assert np.array_equal(ga.view(np.uint32), oa.view(np.uint32)), np.abs(ga - oa).max()


def _perspective_items(org, n, projection):
    import math
    items = []
    for k, (x, y) in enumerate(org):
        if projection == 0:
            th = 0.002 * (k - 1.5)
            H = np.array([[math.cos(th), -math.sin(th), x - 150], [math.sin(th), math.cos(th), 3 * k],
                          [1e-5 * k, -2e-5, 1.0]])
        else:
            f = 500.0
            H = np.array([[1 / f, 0, (x - 150) / f], [0, 1 / f, 0.004 * k], [0, 0, 1]])
        Hi = np.linalg.inv(H)
        items.append((k * 100, 0, k * 100 + 300, 210, list(Hi.ravel())))
    res = 1.0 if projection == 0 else 1 / 500.0
    pmin = (-150.0, -100.0) if projection == 0 else (-0.35, -0.22)
    g = dict(projection=projection, res_x=res, res_y=res, proj_min_x=pmin[0], proj_min_y=pmin[1])
    return items, g


@pytest.mark.parametrize("lazy,ordered", [(1, 0), (1, 1), (0, 0), (0, 1)])
def test_linear_blend_bit_exact(engine, orc, lazy, ordered):
    imgs, org = synth.make_stack(4, 300, 200, 100, 7)
    items, geom = synth.translation_blend_setup(org, 300, 200)
    p = default_params(lazy_read=lazy, ordered_input=ordered)
    a = engine.blend(imgs, items, geom, 0, p)
    b = orc.blend(imgs, items, geom, 0, p)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), np.abs(a - b).max()


@pytest.mark.parametrize("gauss_window_factor", [6, 4, 8])
@pytest.mark.parametrize("bands", [1, 2, 5])
def test_multiband_blend_bit_exact(engine, orc, bands, gauss_window_factor):
    """GAUSS_WINDOW_FACTOR sets the multiband blender's tap count and halo (blend.cu)."""
    imgs, org = synth.make_stack(4, 300, 200, 100, 7)
    items, geom = synth.translation_blend_setup(org, 300, 200)
    p = default_params(multiband=bands, gauss_window_factor=gauss_window_factor)
    a = engine.blend(imgs, items, geom, bands, p)
    b = orc.blend(imgs, items, geom, bands, p)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), np.abs(a - b).max()


@pytest.mark.parametrize("projection", [0, 1, 2])
@pytest.mark.parametrize("bands", [0, 3])
def test_blend_projections_bit_exact(engine, orc, projection, bands):
    imgs, org = synth.make_stack(4, 300, 200, 100, 7)
    items, geom = _perspective_items(org, 4, projection)
    a = engine.blend(imgs, items, geom, bands)
    b = orc.blend(imgs, items, geom, bands)
    assert (a < 0).mean() < 0.9
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), np.abs(a - b).max()


def test_blend_full_size_properties(engine):
    """At a BASELINE shape (1500x1112 crops) the composite of crops of ONE canvas
    must reproduce that canvas where covered: linear blend of identical content is
    the content itself (weights cancel) up to float rounding."""
    imgs, org = synth.config_stack("ordered_13x1500x1112", n=3)
    items, geom = synth.translation_blend_setup(org, 1500, 1112)
    out = engine.blend(imgs, items, geom, 0)
    canvas = synth.make_canvas(1112, 1500 + 500 * 2, 2)[:out.shape[0], :out.shape[1]]
    covered = out[..., 0] >= 0
    assert covered.mean() > 0.95
    assert np.abs(out[covered] - canvas[covered]).max() < 1e-5
    mb = engine.blend(imgs, items, geom, 5)
    cov2 = mb[..., 0] >= 0
    # multiband blurs ROI-border black into the bands (reference behaviour), so only
    # the bulk statistics are a property: range, coverage, small mean error
    assert cov2.mean() > 0.95
    assert mb[cov2].min() >= 0.0 and mb[cov2].max() <= 1.0
    assert np.abs(mb[cov2] - canvas[cov2]).mean() < 5e-3


def test_match_tensor_path_equals_exact_path(engine, orc, monkeypatch, match_mode):
    """The tensor-core nomination + certified exact decisions must give the same pairs
    as the all-fp32 CUDA-core path and as the oracle, including near-threshold
    ratios (heavy noise) where the fp16 scores cannot decide on their own."""
    rng = np.random.RandomState(77)
    a = synth.rootsift_like(1500, 8)
    b = a[rng.permutation(1500)][:1300] + rng.randn(1300, 128).astype(np.float32) * 30.0
    want = orc.match(a, b)
    monkeypatch.delenv("PANO_MATCH_PATH", raising=False)
    got_tc = engine.match_bruteforce(a, b)
    monkeypatch.setenv("PANO_MATCH_PATH", "exact")
    got_ex = engine.match_bruteforce(a, b)
    monkeypatch.delenv("PANO_MATCH_PATH", raising=False)
    assert np.array_equal(got_ex, want)
    assert np.array_equal(got_tc, want)
    assert 50 < len(want) < 1300


@pytest.mark.parametrize("gauss_window_factor", [6, 4, 8])
@pytest.mark.parametrize("bands", [0, 2, 5])
def test_blend_row_strips_equal_full_canvas(engine, bands, gauss_window_factor):
    """pano_blend_rows_dev: uneven row strips (the multi-GPU partition of the canvas) concatenate to
    exactly the mosaic pano_blend_dev produces — for the multiband blender through ROIs clipped to
    the strip plus the summed blur half-widths, which GAUSS_WINDOW_FACTOR sets."""
    imgs, org = synth.make_stack(5, 260, 200, 90, 77, rows=2, step_y=70)
    items, geom = synth.translation_blend_setup(org, 260, 200)
    p = default_params(multiband=bands, lazy_read=0, gauss_window_factor=gauss_window_factor)
    shapes = [im.shape[:2] for im in imgs]
    tw, th = max(it[2] for it in items), max(it[3] for it in items)
    d_imgs = [engine.dev_alloc(im.nbytes) for im in imgs]
    for d, im in zip(d_imgs, imgs):
        engine.dev_upload(d, im)
    d_out = engine.dev_alloc(tw * th * 12)
    full = np.empty((th, tw, 3), np.float32)
    engine.blend_dev(d_imgs, shapes, items, geom, d_out, tw, th, bands, p)
    engine.dev_download(full, d_out)
    cuts = [0, 7, 64, 65, 130, th]                     # strips thinner and thicker than the halo
    parts = []
    for r0, r1 in zip(cuts[:-1], cuts[1:]):
        part = np.empty((r1 - r0, tw, 3), np.float32)
        engine.blend_rows_dev(d_imgs, shapes, items, geom, d_out, tw, th, r0, r1, bands, p)
        engine.dev_download(part, d_out)
        parts.append(part)
    for d in d_imgs + [d_out]:
        engine.dev_free(d)
    got = np.concatenate(parts)
    assert got.tobytes() == full.tobytes()


# ----------------------------------------------------------------------------- matcher edges
# The inputs come from tests/test_match_bound.py, whose CPU model checks tc_eps on the same sets.
from tests import test_match_bound as mb  # noqa: E402


def _match_both_ways(engine, orc, monkeypatch, a, b, params=None):
    """a x b and b x a on the tensor path and on the exact fp32 path, each against the oracle."""
    want = [orc.match(a, b, params), orc.match(b, a, params)]
    for path in (None, "exact"):
        if path:
            monkeypatch.setenv("PANO_MATCH_PATH", path)
        else:
            monkeypatch.delenv("PANO_MATCH_PATH", raising=False)
        got = [engine.match_bruteforce(a, b, params), engine.match_bruteforce(b, a, params)]
        for g, w, d in zip(got, want, ("ab", "ba")):
            assert np.array_equal(g, w), (path, d, len(g), len(w))
    monkeypatch.delenv("PANO_MATCH_PATH", raising=False)
    return want


@pytest.mark.parametrize("ratio", [0.5, 0.6, 0.9, 0.95, 1.0])
def test_match_ratios(engine, orc, monkeypatch, match_mode, ratio):
    """MATCH_REJECT_NEXT_RATIO (refine_row's skip rule, every interval test of k_match_decide), on targets
    with noise from 60 down to 10.  The first 150 targets come twice, so their rows tie exactly
    (min == next_min): ratio 1.0 accepts those whose column test passes too."""
    rng = np.random.RandomState(31)
    a = synth.rootsift_like(400, 31)
    level = np.linspace(60, 10, 320).astype(np.float32)[:, None]
    noisy = a[rng.permutation(400)][:320] + rng.randn(320, 128).astype(np.float32) * level
    b = np.concatenate([noisy[:150], noisy[:150], noisy[150:]])
    want = _match_both_ways(engine, orc, monkeypatch, a, b, default_params(match_reject_next_ratio=ratio))
    assert len(want[0]) > (150 if ratio == 1.0 else 40)


EDGE_SIZES = [127, 128, 129, 255, 256, 257, 383, 385, 511, 512, 513]


@pytest.mark.parametrize("n,m", list(zip(EDGE_SIZES, EDGE_SIZES[5:] + EDGE_SIZES[:5])))
def test_match_block_edges(engine, orc, monkeypatch, match_mode, n, m):
    """Set sizes at the edges of the 128-row query blocks, 256-row target tiles and 64-row exact tiles."""
    a, b = mb.random_rows(n, m, n + m)
    want = _match_both_ways(engine, orc, monkeypatch, a, b)
    assert len(want[0]) > min(n, m) // 10


@pytest.mark.parametrize("scale", mb.SCALES)
def test_match_scaled_descriptors(engine, orc, monkeypatch, match_mode, scale):
    """Descriptor norms other than 512 (DESC_INT_FACTOR): the fp16 scale s and tc_eps follow the norm."""
    a, b = mb.scaled_rows(scale)
    want = _match_both_ways(engine, orc, monkeypatch, a, b)
    assert len(want[0]) > 20


def _match_pairs_both_paths(engine, orc, monkeypatch, fs, sets, pairs, params=None):
    """match_pairs on the tensor path and on the exact fp32 path, every pair against the oracle."""
    want = [orc.match(sets[i], sets[j], params) for i, j in pairs]
    for path in (None, "exact"):
        if path:
            monkeypatch.setenv("PANO_MATCH_PATH", path)
        else:
            monkeypatch.delenv("PANO_MATCH_PATH", raising=False)
        for (i, j), g, w in zip(pairs, engine.match_pairs(fs, pairs, params), want):
            assert np.array_equal(g, w), (path, i, j, len(g), len(w))
    monkeypatch.delenv("PANO_MATCH_PATH", raising=False)
    return want


def test_match_mixed_norms_one_featureset(engine, orc, monkeypatch, match_mode):
    """k_tc_maxnorm takes one maximum over the whole feature set: a norm-2 image is matched at the
    scale of a norm-512 one."""
    sets = mb.mixed_rows()
    fs = engine.featureset_upload(sets)
    pairs = [(0, 1), (1, 0), (2, 3), (3, 2), (0, 2), (2, 0), (3, 1), (1, 3)]
    want = _match_pairs_both_paths(engine, orc, monkeypatch, fs, sets, pairs)
    fs.free()
    assert len(want[2]) > 20


@pytest.mark.parametrize("factor", [100, 4096])
def test_match_sift_features_other_desc_int_factor(engine, orc, monkeypatch, match_mode, factor):
    imgs, _ = synth.make_stack(3, 360, 270, 120, 43)
    p = default_params(desc_int_factor=factor)
    fs = engine.sift_detect_batch(imgs, p)
    descs = [fs.download(i)[1] for i in range(3)]
    pairs = [(0, 1), (1, 0), (1, 2), (2, 1), (2, 0), (0, 2)]
    want = _match_pairs_both_paths(engine, orc, monkeypatch, fs, descs, pairs, p)
    fs.free()
    assert sum(len(w) for w in want) > 30


def test_match_adversarial_fp16_rounding(engine, orc, monkeypatch, match_mode):
    """Rows whose fp16 rounding errors all have one sign (scores down to ~-1), exact duplicates,
    near-duplicates across fp16 midpoints, permutations, and the ratio trap that a bound below ~40% of
    tc_eps decides wrongly."""
    a, b = mb.adversarial_rows(48, 2)
    want = _match_both_ways(engine, orc, monkeypatch, a, b)
    assert len(want[0]) > 40


@pytest.mark.parametrize("parts,block_cap", [("2", None), ("3", None), ("8", None), (None, "1")])
def test_match_adversarial_split_and_fallback(engine, orc, monkeypatch, match_mode, parts, block_cap):
    """The adversarial rows under PANO_MATCH_PARTS column ranges (among 8200 far targets, so that 8 parts
    keep 4 tiles each) and with PANO_MATCH_BLOCK_CAP=1 (every requested row re-scanned in full)."""
    a, b = mb.adversarial_rows(48, 5)
    far = (synth.rootsift_like(8200, 14) * np.float32(0.99)).astype(np.float32)
    b = np.concatenate([far[:4000], b, far[4000:]])
    for k, v in (("PANO_MATCH_PARTS", parts), ("PANO_MATCH_BLOCK_CAP", block_cap)):
        if v:
            monkeypatch.setenv(k, v)
    got = [engine.match_bruteforce(a, b), engine.match_bruteforce(b, a)]
    monkeypatch.delenv("PANO_MATCH_PARTS", raising=False)
    monkeypatch.delenv("PANO_MATCH_BLOCK_CAP", raising=False)
    assert np.array_equal(got[0], orc.match(a, b))
    assert np.array_equal(got[1], orc.match(b, a))
    assert len(got[0]) > 40
