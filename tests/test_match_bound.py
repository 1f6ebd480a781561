"""CPU model of the tensor matcher's fp16 certification (match_tc.cu, match.cu: tc_eps).

k_tc_prep turns every descriptor x into fp16 operands: query form [s*x | 1, 1, n_hi, n_lo, 1], target
form [-2*s*x | n_hi, n_lo, 1, 1, 1], with n = s^2*|x|^2 split into two fp16 halves and s the power of two
that makes the largest n of the whole feature set <= 1024.  The wgmma score q.t is an approximation of
s^2*|xq - xt|^2 + 1; match.cu turns its truncated key back into a squared distance and trusts it only
within tc_eps(|xq|^2, max |x|^2).  This file rebuilds those operands in numpy, takes the exact float64
dot product of the fp16 operands, widens it by a bound on any fp32 accumulation order (the wgmma
summation order is unspecified), applies the 0xffffff00 key truncation, and checks that every
reachable approximate distance lies within tc_eps of the exact fp32 distance of feature/dist.cc's SSE
order (what the oracle and the exact kernels compute).

The generators here are also the inputs of the GPU matcher tests (tests/test_gpu_match_warp_blend.py)."""
import numpy as np
import pytest

from openpano_b200 import synth

F32 = np.float32
KEY_MASK = np.uint32(0xffffff00)


# ----------------------------------------------------------------------------- the device's operands
def row_norms(x):
    """k_tc_maxnorm: |x|^2 in fp32, one running sum over the 128 components in order."""
    x = np.asarray(x, F32)
    acc = np.zeros(len(x), F32)
    for k in range(128):
        acc = acc + x[:, k] * x[:, k]
    return acc


def tc_scale(maxn2):
    """tc_scale_from_maxnorm: s = 2^-e, e = ceil(log2(maxn2 / 1024) / 2), in fp32."""
    maxn2 = F32(maxn2)
    if not maxn2 > 0:
        return F32(1.0)
    e = int(np.ceil(F32(0.5) * np.log2(maxn2 / F32(1024.0))))
    return F32(2.0 ** -e)


def tc_operands(x, norms, s):
    """(query rows, target rows) of k_tc_prep as float64 copies of the fp16 values, K = 133."""
    x = np.asarray(x, F32)
    q = (x * s).astype(np.float16)
    t = (x * F32(-2.0 * s)).astype(np.float16)
    n = norms * s * s
    nh = n.astype(np.float16)
    nl = (n - nh.astype(F32)).astype(np.float16)
    one = np.ones(len(x), np.float16)
    qx = np.concatenate([q, np.stack([one, one, nh, nl, one], 1)], 1)
    tx = np.concatenate([t, np.stack([nh, nl, one, one, one], 1)], 1)
    return qx.astype(np.float64), tx.astype(np.float64)


def tc_eps(nq, nmax):
    """match.cu tc_eps in fp32 (the library is built without FMA contraction)."""
    return F32(0.00215) * np.sqrt(F32(nq) * F32(nmax)) + F32(0.0005) * F32(nmax) + F32(1.0)


def exact_d2(a, b):
    """feature/dist.cc's SSE branch: four lane accumulators over 32 steps, (l0 + l1) + (l2 + l3)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    out = np.empty((len(a), len(b)), F32)
    for r0 in range(0, len(a), 64):
        d = (a[r0:r0 + 64, None, :] - b[None, :, :]).reshape(-1, len(b), 32, 4)
        lanes = np.zeros(d.shape[:2] + (4,), F32)
        for k in range(32):
            lanes = lanes + d[:, :, k] * d[:, :, k]
        out[r0:r0 + 64] = (lanes[..., 0] + lanes[..., 1]) + (lanes[..., 2] + lanes[..., 3])
    return out


def _key_to_d2(v, s):
    """A reachable fp32 score -> the packed key with its low 8 bits cleared -> (key - 1) / s^2 in fp32."""
    key = (np.asarray(v, F32).view(np.uint32) & KEY_MASK).view(F32)
    return (key - F32(1.0)) * F32(1.0 / (float(s) * float(s)))


def model(sets, pairs):
    """For each (i, j) in pairs: the score range of every row of sets[i] against every row of sets[j], its
    extreme approximate distances, the exact fp32 distances and tc_eps, with s from the whole set."""
    norms = [row_norms(x) for x in sets]
    nmax = max((float(n.max()) for n in norms if len(n)), default=0.0)
    s = tc_scale(nmax)
    ops = [tc_operands(x, n, s) for x, n in zip(sets, norms)]
    out = []
    for i, j in pairs:
        q, t = ops[i][0], ops[j][1]
        score = q @ t.T
        # any fp32 summation order of the 133 products stays within 145 * 2^-24 * sum |products|
        err = 145.0 * 2.0 ** -24 * (np.abs(q) @ np.abs(t).T)
        lo = (score - err).astype(F32)
        hi = (score + err).astype(F32)
        lo = np.where(lo > score - err, np.nextafter(lo, F32(-np.inf)), lo)
        hi = np.where(hi < score + err, np.nextafter(hi, F32(np.inf)), hi)
        # truncation and (key - 1) / s^2 are monotone, so the reachable approximations lie between these two
        ap_lo, ap_hi = _key_to_d2(lo, s), _key_to_d2(hi, s)
        out.append(dict(score=score, lo=lo, hi=hi, ap_lo=ap_lo, ap_hi=ap_hi, d2=exact_d2(sets[i], sets[j]),
                        eps=tc_eps(norms[i][:, None], nmax), s=s, nq=norms[i], nmax=nmax))
    return out


# ----------------------------------------------------------------------------- inputs
def midpoint_rows(v, up, s):
    """fp32 rows x whose scaled components s*x sit one fp32 ulp above (up[row]) or below the fp16
    rounding midpoint just above the scaled target values v, so that k_tc_prep rounds every component
    of a row up, or every one down, by half an fp16 ulp."""
    v = np.asarray(v, np.float64)
    lo = v.astype(np.float16)
    lo = np.where(lo.astype(np.float64) > v, np.nextafter(lo, np.float16(0)), lo)
    mid = (lo.astype(F32) + np.nextafter(lo, np.float16(np.inf)).astype(F32)) * F32(0.5)
    x = np.where(np.asarray(up)[:, None], np.nextafter(mid, F32(np.inf)), np.nextafter(mid, F32(0)))
    return (x / F32(s)).astype(F32)


def _patterns(n, rng):
    """Scaled rows (s = 1/16) of 42 components at 4 and 86 at 2: the largest relative fp16 rounding
    error (half an ulp just above a power of two) at a scaled squared norm of ~1018 <= 1024."""
    v = np.full((n, 128), 2.0)
    for r in range(n):
        v[r, rng.choice(128, 42, replace=False)] = 4.0
    return v


def adversarial_rows(n, seed):
    """(queries, targets) of norm <= 512 (s = 1/16) whose scaled components sit just above or just below
    fp16 midpoints, so that the fp16 rounding errors of a row all have one sign and do not cancel.
    Per query: an exact duplicate, the same row rounded the other way (every component moved across its
    midpoint: exact distance ~0, approximate distance off by ~500), a copy with three components moved
    by 1e-3, a copy with four components permuted, and a pair (T1, T2) built so that the approximate
    distances misstate the second-best by nearly tc_eps: q and T2 round down, T1 rounds up, and the
    exact distances sit just past the ratio test (|q - T1|^2 = 0.64 |q - T2|^2 + 80), which a bound
    of under ~40% of tc_eps would wrongly accept at ratio 0.8."""
    rng = np.random.RandomState(seed)
    s = 1.0 / 16
    v = _patterns(n, rng)
    up = rng.rand(n) < 0.5
    q = midpoint_rows(v, up, s)
    targets = [q.copy(), midpoint_rows(v, ~up, s)]
    moved = q.copy()
    for r in range(n):
        moved[r, rng.choice(128, 3, replace=False)] += F32(1e-3)
    targets.append(moved)
    perm = q.copy()
    for r in range(n):
        c = rng.choice(128, 4, replace=False)
        perm[r, c] = perm[r, np.roll(c, 1)]
    targets.append(perm)
    # the ratio trap: component 0 / 1 lowered (norm stays <= 512) so that D1 = 0.64 D2 + 80 with D2 = 2000
    vt = _patterns(n, rng)
    trap_q = midpoint_rows(vt, np.zeros(n, bool), s)
    d2, d1 = 2000.0, 0.64 * 2000.0 + 80.0
    v1, v2 = vt.copy(), vt.copy()
    v1[:, 0] -= np.sqrt(d1) * s
    v2[:, 1] -= np.sqrt(d2) * s
    t1 = midpoint_rows(v1, np.ones(n, bool), s)
    t2 = midpoint_rows(v2, np.zeros(n, bool), s)
    # the trap queries have patterns of their own: every other target sits far from them
    a = np.concatenate([q, trap_q])
    b = np.concatenate(targets + [t1, t2])
    order = rng.permutation(len(b))
    return a, b[order]


def random_rows(n, m, seed, noise=38.0):
    rng = np.random.RandomState(seed)
    a = synth.rootsift_like(max(n, m), seed)
    b = a[rng.permutation(len(a))][:m] + rng.randn(m, 128).astype(F32) * F32(noise)
    return a[:n], b


SCALES = [2.0 ** -8, 1.0 / 512, 100.0 / 512, 8.0]       # 8 = 4096 / 512: DESC_INT_FACTOR 4096


def scaled_rows(scale, seed=3):
    a, b = random_rows(300, 260, seed)
    return (a * F32(scale)).astype(F32), (b * F32(scale)).astype(F32)


def mixed_rows(seed=4):
    """A norm-512 image and a norm-2 image in one feature set: s comes from the largest norm of all."""
    a, b = random_rows(300, 260, seed)
    tiny_a, tiny_b = random_rows(200, 180, seed + 1)
    return [a, b, (tiny_a * F32(2.0 ** -8)).astype(F32), (tiny_b * F32(2.0 ** -8)).astype(F32)]


SETS = {
    "random": lambda: list(random_rows(300, 260, 1)),
    "adversarial": lambda: list(adversarial_rows(48, 2)),
    **{f"scaled_{sc:g}": (lambda sc=sc: list(scaled_rows(sc))) for sc in SCALES},
    "mixed": mixed_rows,
}


# ----------------------------------------------------------------------------- tests
@pytest.mark.parametrize("name", list(SETS))
def test_tc_eps_bounds_every_approximation(name):
    sets = SETS[name]()
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets))]
    worst = 0.0
    for m in model(sets, pairs):
        dev = np.maximum(np.abs(m["ap_lo"].astype(np.float64) - m["d2"]), np.abs(m["ap_hi"].astype(np.float64) - m["d2"]))
        assert (dev <= m["eps"]).all(), (name, float((dev - m["eps"]).max()))
        worst = max(worst, float((dev / m["eps"]).max()))
        # every upper bound built from a nominated score stays positive (refine_row: mn_hi, sec_hi = m + eps),
        # so no row is rejected on bounds alone while its approximate minimum is still below zero
        assert (m["ap_lo"] + m["eps"] > 0).all(), name
    if name == "adversarial":
        assert worst > 0.7, worst          # the adversarial rows get close to the bound ...
    if name == "random":
        assert worst < 0.2, worst          # ... random RootSIFT-like rows stay far inside it


def test_lowest_reachable_score():
    """Scores are not >= 1: s^2 |x|^2 - sum fp16(s x_i)^2 reaches -n/1024 per row, so a row against
    itself scores down to 1 - n/512, i.e. -1 at n = 1024 (here ~-0.98).  The fp32 keys of negative scores
    order backwards as signed ints; test_tc_eps_bounds_every_approximation shows the bounds hold anyway."""
    a, b = adversarial_rows(48, 2)
    ms = model([a, b], [(0, 0), (0, 1)])
    low = min(float(m["score"].min()) for m in ms)
    assert -1.0 <= low < -0.95, low
    n = ms[0]["nq"] * ms[0]["s"] * ms[0]["s"]
    floor = 1.0 - 2.0 * n.astype(np.float64) * (2.0 ** -10 + 2.0 ** -22) - 1e-4
    assert (np.diagonal(ms[0]["score"]) >= floor).all()
    # random RootSIFT-like rows never get near zero
    a, b = random_rows(300, 260, 1)
    assert float(model([a, b], [(0, 0)])[0]["score"].min()) > 0.9


def test_ratio_trap_needs_the_full_bound():
    """The trap rows of adversarial_rows: with tc_eps the second-best interval holds the exact distance;
    with the bound's first coefficient lowered to 0.0005 it misses it by ~250, and refine_row would call
    the argmin certain and the ratio test (0.8) an accept the reference rejects."""
    a, b = adversarial_rows(48, 2)
    m = model([a, b], [(0, 1)])[0]
    traps = np.arange(48, 96)
    d2 = m["d2"][traps].astype(np.float64)
    best = d2.argmin(1)
    for r, k in enumerate(traps):
        row = d2[r]
        j1 = best[r]
        j2 = np.argsort(row)[1]
        assert row[j1] > 0.64 * row[j2]                             # the reference rejects
        m1, m2 = float(m["ap_hi"][k, j1]), float(m["ap_lo"][k, j2])
        eps, nq, nmax = float(m["eps"][k, 0]), float(m["nq"][k]), m["nmax"]
        weak = 0.0005 * np.sqrt(nq * nmax) + 0.0005 * nmax + 1.0
        assert m2 - m1 > 2 * weak and row[j1] <= 0.64 * (m2 - weak)  # the weak bound: certain, accepted
        assert not (m2 - m1 > 2 * eps)                              # tc_eps: uncertain, re-scanned exactly


def test_reversed_negative_keys_keep_decisions():
    """Negative scores order backwards as signed-int keys, so the nominated (m1, m2) of a row j may be its
    two LARGEST negative-score approximations, with m2 < m1.  refine_row then finds the argmin uncertain
    and gives j the bounds [max(m1 - eps, 0), m1 + eps] and [max(m2 - eps, 0), m2 + eps]; k_match_decide
    uses sec_hi = m2 + eps as column j's bound on min_{kk != k} d(j, kk), which is below the truth when k is
    the column behind m2.  This checks, for the scores at both ends of their reachable range, that
    (1) that too-low bound never rejects a row k the reference accepts: d(j, k) > R * (m2 + eps) implies
    d(j, k) > R * min_{kk != k} d(j, kk) for every ratio R <= 1, and (2) the filter threshold m2 + 2.5 eps
    (k_tc_gather_rows) covers every column that can be j's exact best or second best."""
    a, b = adversarial_rows(48, 2)
    m = model([a, b], [(0, 1)])[0]
    d2 = m["d2"].astype(np.float64)
    eps = m["eps"][:, 0].astype(np.float64)
    rows = np.arange(len(d2))
    order = np.argsort(d2, axis=1, kind="stable")
    top2 = d2[rows, order[:, 1]]
    reversed_rows = 0
    for v in (m["lo"], m["hi"]):
        key = (v.view(np.uint32) & KEY_MASK).view(np.int32)
        ap = _key_to_d2(v, m["s"]).astype(np.float64)
        nom = np.argsort(key, axis=1, kind="stable")[:, :2]            # the kernel's signed-key top-2
        m1, m2 = ap[rows, nom[:, 0]], ap[rows, nom[:, 1]]
        reversed_rows += int((m2 < m1).sum())
        # min over kk != k of d(j, kk): the row minimum, or its second value where k is the argmin
        others = np.where(np.arange(d2.shape[1])[None, :] == order[:, :1], top2[:, None], d2[rows, order[:, 0]][:, None])
        for ratio in (0.5, 0.6, 0.8, 0.9, 0.95, 1.0):
            low_bound_rejects = d2 > ratio * (m2 + eps)[:, None]
            assert (d2[low_bound_rejects] > ratio * others[low_bound_rejects]).all(), ratio
        thr = m2 + 2.5 * eps
        for c in (order[:, 0], order[:, 1]):
            assert (m["ap_hi"][rows, c] <= thr).all()
    assert reversed_rows > 0            # the case occurs on these rows
