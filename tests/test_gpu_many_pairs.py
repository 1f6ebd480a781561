"""GPU parity of the pair-indexed entry points at unordered-mosaic pair counts: the matcher over all
79,800 pairs of 400 feature sets (and prefixes at the 32,768 / 65,536 grid edges), RANSAC scoring and
bundle adjustment over 65,535, 65,536 and 70,000 pairs, each bit for bit against the oracle.  The
reference's unordered mode matches every pair of images (stitcher.cc:98-100), so 257 images already
give 32,896 pairs.  Sizes per pair stay tiny: the counts are what is tested.  Also: every image-count
limit the header states is refused with PANO_ERR_INVALID, and the context keeps working."""
import ctypes as C

import numpy as np
import pytest

from openpano_b200 import synth
from openpano_b200.capi import LIB, PanoError
from tests import ba_step_util as bs
from tests import golden_util as gu
from tests.ba_util import ba_case
from tests.ransac_util import ransac_case

pytestmark = pytest.mark.gpu

PANO_ERR_INVALID = -2
N_SETS = 400
EDGES = (32767, 32768, 65535, 65536)


# ------------------------------------------------------------------ matcher

@pytest.fixture(scope="module")
def match_case(orc):
    """400 ragged feature sets drawn from one pool of 240 RootSIFT-like rows plus per-set noise, so that
    two sets sharing pool rows match; sizes 0, 1 and up to 40; some sets hold exact duplicate rows (ties).
    -> (sets, pairs [79800, 2] in all-pairs order, expected match list per pair)."""
    rng = np.random.RandomState(2024)
    pool = synth.rootsift_like(240, 77)
    sets = []
    for s in range(N_SETS):
        n = [0, 1, 40][s] if s < 3 else int(rng.randint(0, 41))
        rows = pool[rng.choice(len(pool), n, replace=True)] + rng.randn(n, 128).astype(np.float32) * 6.0
        if n >= 4 and s % 7 == 0:
            rows[n - 1] = rows[0]                       # exact duplicate: zero-distance tie inside the set
        sets.append(np.ascontiguousarray(rows, np.float32))
    iu = np.triu_indices(N_SETS, 1)
    pairs = np.stack(iu, 1).astype(np.int32)
    flip = rng.rand(len(pairs)) < 0.5                   # both orders of (i, j): MatchData::reverse either way
    pairs[flip] = pairs[flip][:, ::-1]
    assert len(pairs) == 79800
    want = [orc.match(sets[i], sets[j]) for i, j in pairs]
    return sets, pairs, want


@pytest.fixture(params=["tensor_lazy0", "tensor_lazy1", "exact"])
def match_path(request, monkeypatch):
    monkeypatch.delenv("PANO_MATCH_PATH", raising=False)
    if request.param == "exact":
        monkeypatch.setenv("PANO_MATCH_PATH", "exact")
        monkeypatch.delenv("PANO_MATCH_LAZY", raising=False)
    else:
        monkeypatch.setenv("PANO_MATCH_LAZY", request.param[-1])
    return request.param


def _check_lists(got, want):
    assert len(got) == len(want)
    bad = [k for k, (g, w) in enumerate(zip(got, want)) if not np.array_equal(g, w)]
    assert not bad, (len(bad), bad[:5])


def test_match_all_pairs_of_400_sets(engine, match_case, match_path):
    """pano_match_pairs, pano_match_pairs_dev and three row shards over all 79,800 pairs."""
    sets, pairs, want = match_case
    total = sum(len(w) for w in want)
    assert total > 5000                                 # not vacuous: thousands of accepted rows
    assert sum(len(w) > 0 for w in want) > 10000
    fs = engine.featureset_upload(sets)
    try:
        got = engine.match_pairs(fs, pairs)
        _check_lists(got, want)
        assert sum(len(g) for g in got) == total
        assert engine.match_pairs_dev(fs, pairs) == total
        S = 3
        parts = [engine.match_pairs(fs, pairs, shard=(s, S)) for s in range(S)]
        _check_lists([np.concatenate([p[k] for p in parts]) for k in range(len(pairs))], want)
        assert sum(engine.match_pairs_dev(fs, pairs, shard=(s, S)) for s in range(S)) == total
    finally:
        fs.free()


@pytest.mark.parametrize("n_pairs", EDGES)
def test_match_pair_count_edges(engine, match_case, match_path, n_pairs):
    """Prefixes that end one below and one at the 32,768-pair (two sides per pair) and 65,536-pair limits."""
    sets, pairs, want = match_case
    fs = engine.featureset_upload(sets)
    try:
        got = engine.match_pairs(fs, pairs[:n_pairs])
        _check_lists(got, want[:n_pairs])
        assert engine.match_pairs_dev(fs, pairs[:n_pairs]) == sum(len(w) for w in want[:n_pairs])
    finally:
        fs.free()


# ------------------------------------------------------------------ RANSAC scoring

def _ransac_pool():
    """Distinct small cases (0-30 matches, 0-8 hypotheses) and the special ones; pair k uses case k % len."""
    rng = np.random.RandomState(31)
    pool = []
    for q in range(251):
        pool.append(ransac_case(int(rng.randint(0, 31)), int(rng.randint(0, 9)), 1000 + q))
    kp1, kp2, homos, thres = ransac_case(30, 6, 7)
    pool.append((kp1, kp2, np.zeros((0, 9)), thres))                       # no hypotheses
    pool.append((np.zeros((0, 2)), np.zeros((0, 2)), homos, thres))        # no matches
    true_h = np.array([1.0, 0.02, 480.0, -0.015, 1.0, 6.0, 1e-5, -2e-5, 1.0])
    far = homos + np.array([0, 0, 300.0, 0, 0, 300.0, 0, 0, 0])
    pool.append((kp1, kp2, np.stack([far[0], true_h, far[1], true_h]), thres))   # tie between 1 and 3
    pool.append((kp1, kp2, np.concatenate([far[:5], true_h[None]]), thres))      # the last one is the best
    return pool


@pytest.fixture(scope="module")
def ransac_expect(orc):
    pool = _ransac_pool()
    want = [orc.ransac_score(*c) for c in pool]
    tie, last = want[-2], want[-1]
    assert tie[2][1] == tie[2][3] > 0 and tie[0] == 1                    # the oracle's first maximum
    assert last[0] == 5 and last[1] > max(last[2][:5])
    return pool, want


@pytest.mark.parametrize("n_pairs", [65535, 65536, 70001])
def test_ransac_many_pairs(engine, ransac_expect, n_pairs):
    pool, want = ransac_expect
    L = len(pool)
    idx = [k % L for k in range(n_pairs)]
    idx[-1] = L - 1                                     # the last pair of the call: its last hypothesis wins
    idx[-2] = L - 2
    got = engine.ransac_score_pairs([pool[q] for q in idx])
    bad = []
    for k, q in enumerate(idx):
        g, w = got[k], want[q]
        if not (g[0] == w[0] and g[1] == w[1] and np.array_equal(g[2], w[2]) and np.array_equal(g[3], w[3])):
            bad.append(k)
    assert not bad, (len(bad), bad[:5])
    assert sum(g[1] for g in got) > n_pairs              # inliers are found, not just empty pairs


# ------------------------------------------------------------------ bundle adjustment

@pytest.fixture(scope="module")
def ba_repeated(orc):
    """The golden 5-camera problem's 7 pairs (and their matrices) repeated, 1-4 points per pair; the
    coordinates are the golden problem's points taken in turn.  Repeated and reversed camera pairs are
    valid inputs.  -> n -> (pairs, mats, hto, pts, oracle rows, oracle J^T J) of n pairs."""
    g, gs = gu.load("ba_5cams.npz"), gu.load("ba_step_5cams.npz")
    _, base_pairs, base_pts = ba_case(5, 40, 5, extra_pairs=3)
    assert gu.same_bits(g["mats"], gs["mats"])
    assert any(f > t for f, t, _ in base_pairs) and any(f < t for f, t, _ in base_pairs)
    cache = {}

    def make(n):
        if n not in cache:
            rng = np.random.RandomState(n)
            counts = rng.randint(1, 5, n)
            pairs = [(base_pairs[k % 7][0], base_pairs[k % 7][1], int(counts[k])) for k in range(n)]
            mats = g["mats"][np.arange(n) % 7]
            hto = gs["hto"][np.arange(n) % 7]
            pts = base_pts[np.arange(int(counts.sum())) % len(base_pts)]
            cache[n] = (pairs, mats, hto, pts) + orc.ba_jacobian(5, pairs, mats, pts[:, :2])
        return cache[n]
    return make


@pytest.mark.parametrize("n_pairs", [65535, 65536, 70001])
def test_ba_jacobian_many_pairs(engine, ba_repeated, n_pairs):
    pairs, mats, _, pts, want_rows, want_jtj = ba_repeated(n_pairs)
    rows, jtj = engine.ba_jacobian(5, [(f, t, n, m) for (f, t, n), m in zip(pairs, mats)], pts[:, :2])
    assert gu.same_bits(rows, want_rows)
    assert gu.same_bits(jtj, want_jtj)


@pytest.mark.parametrize("n_pairs", [65535, 65536, 70001])
def test_ba_session_many_pairs(engine, ba_repeated, n_pairs):
    pairs, mats, hto, pts, w_rows, w_jtj = ba_repeated(n_pairs)
    w_res, w_avg, w_max = bs.orc_error(pairs, hto, pts)
    w_b = bs.orc_jtr(5, pairs, w_rows, w_res)
    s = engine.ba_session(5, pairs, pts)
    try:
        avg, mx, res = s.error(hto)
        assert gu.same_bits(res, w_res)
        assert gu.same_bits(np.float64(avg), np.float64(w_avg)) and gu.same_bits(np.float64(mx), np.float64(w_max))
        jtj, b, rows = s.normal_equations(mats, want_rows=True)
        assert gu.same_bits(rows, w_rows) and gu.same_bits(jtj, w_jtj) and gu.same_bits(b, w_b)
    finally:
        s.close()


# ------------------------------------------------------------------ limits kept on purpose

def _refused(call):
    """The call is refused as a bad argument that names the limit, not as a failed launch."""
    with pytest.raises(PanoError) as e:
        call()
    assert e.value.code == PANO_ERR_INVALID and "limit" in str(e.value), e.value


def _still_works(engine):
    a = synth.rootsift_like(50, 3)
    b = a[::-1] + np.float32(1.0)
    got = engine.match_bruteforce(a, b)
    assert len(got) == 50


def test_image_count_limits_are_refused(engine):
    n = 65536
    # featureset: its tensor-core operands are prepared per image on gridDim.y
    _refused(lambda: engine.featureset_upload([np.zeros((0, 128), np.float32)] * n))
    _still_works(engine)
    d = engine.dev_alloc(4096)
    try:
        # 8-bit -> f32 conversion batch (images on gridDim.y)
        _refused(lambda: engine.rgb8_to_mat32f_batch_dev([d] * n, [4] * n, [4] * n, [3] * n, [d] * n))
        _still_works(engine)
        # cylinder warp batch (images on gridDim.z)
        _refused(lambda: engine.cyl_warp_batch_dev([d] * n, [(4, 4)] * n, [d] * n))
        _still_works(engine)
    finally:
        engine.dev_free(d)
    # blend: images on gridDim.z of the multi-band first level
    _, org = synth.make_stack(2, 16, 12, 4, 1)
    items, geom = synth.translation_blend_setup(org, 16, 12)
    _refused(lambda: engine.blend_stream([(12, 16)] * n, [items[0]] * n, geom, bands=2))
    _still_works(engine)
    # bundle adjustment: J^T J blocks on (camera, camera).  Called directly: the binding would allocate
    # the (6n)^2 J^T J output on the host first.
    jtj = np.zeros(1, np.float64)
    _refused(lambda: engine._check(LIB.pano_ba_jacobian(engine._h, n, 0, None, None, None,
                                                        jtj.ctypes.data_as(C.POINTER(C.c_double)))))
    _refused(lambda: engine.ba_session(n, [], np.zeros((0, 4))))
    _still_works(engine)
