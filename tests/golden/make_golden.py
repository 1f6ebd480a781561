#!/usr/bin/env python
"""Generates tests/golden/*.npz from the REFERENCE's own translation units
(oracle/_ref/libopenpano_ref.so, built by oracle/Makefile from the reference's
src/ with -O2 -ffp-contract=off -msse3, single thread).

The reference ships no golden vectors for this path (SURVEY.md §4), so these
fixtures ARE the pin: the plain-C oracle and the CUDA engine are both compared
against them bit for bit.  Inputs come from openpano_b200.synth (seeded numpy);
each fixture stores a SHA-256 of its inputs so generator drift is detected.

Run where the reference tree was available at build time (oracle/_ref built):
    python tests/golden/make_golden.py [imgio | ba | vs_ref]
"""
import hashlib
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))

from openpano_b200 import synth  # noqa: E402
from openpano_b200._abi import default_params  # noqa: E402
from tests.checker import get_checker  # noqa: E402

OUT = Path(__file__).resolve().parent


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def plane_crc(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()[:8], np.uint64).copy()


def imgio(ref):
    """read_img / crop / write_rgb through the reference's own lib/imgio.cc + lib/imgproc.cc."""
    from tests.golden_util import imgio_inputs
    pix, grey, mos = imgio_inputs()
    rect, cropped = ref.crop(mos)
    np.savez_compressed(OUT / "imgio.npz", input_sha=np.array(sha(pix, grey, mos)),
                        read_rgb=ref.read_img_rgb8(pix), read_grey=ref.read_img_rgb8(grey),
                        crop_wh=rect[2:], cropped=cropped, write_full=ref.write_rgb8(mos),
                        write_cropped=ref.write_rgb8(cropped))
    print("imgio: crop", rect, cropped.shape)


def ba(ref):
    """The reference's own calcJacobianSymbolic (incremental_bundle_adjuster.cc:276-385) and the per-pair
    matrices, evaluated by the reference's own Homography / Camera operations (oracle/refshim/ref_ba.cc)."""
    from tests.ba_util import ba_case
    cams, pairs, pts = ba_case(5, 40, 5, extra_pairs=3)
    mats = ref.ba_pair_mats(cams, pairs)
    rows, jtj = ref.ba_jacobian_ref(cams, pairs, pts)
    np.savez_compressed(OUT / "ba_5cams.npz", input_sha=np.array(sha(cams, np.array(pairs), pts)),
                        mats=mats, rows=rows, jtj=jtj)
    print("ba:", len(pairs), "pairs,", len(pts), "matches")


_RATIO_SCRIPT = """
import json, sys
sys.path.insert(0, {root!r})
from tests.checker import get_checker
from tests import test_oracle_vs_ref as t
print(json.dumps(t.digests(t.case_match_other_ratios(get_checker('ref'), {ratio!r}))))
"""


def vs_ref(ref):
    """Digests of the reference's outputs for every case of tests/test_oracle_vs_ref.py, and the
    per-pair matrices its bundle-adjustment cases start from."""
    import json
    import subprocess
    from tests import test_oracle_vs_ref as t
    from tests.ba_util import ba_case
    res = {key: np.array(t.digests(fn(ref, *args))) for key, fn, args in t.golden_cases()}
    for ratio, _, _ in t.MATCH_RATIOS:       # one process per ratio: the reference freezes it on first use
        out = subprocess.run([sys.executable, "-c", _RATIO_SCRIPT.format(root=str(ROOT), ratio=ratio)],
                             capture_output=True, text=True, check=True)
        res[t.case_key("test_match_other_ratios", ratio)] = np.array(json.loads(out.stdout.strip().splitlines()[-1]))
    for args in t.BA_CASES:
        n_cam, per_pair, seed, extra = args
        cams, pairs, pts = ba_case(n_cam, per_pair, seed, extra_pairs=extra)
        res[t.ba_mats_key(*args)] = ref.ba_pair_mats(cams, pairs)
        res[t.case_key("test_ba_jacobian", *args)] = np.array(t.digests(ref.ba_jacobian_ref(cams, pairs, pts)))
    np.savez_compressed(OUT / t.FIXTURE, **res)
    print("vs_ref:", len(res), "entries")


def main():
    ref = get_checker("ref")
    assert ref.num_threads() == 1
    if sys.argv[1:] == ["imgio"]:      # add this fixture without rewriting the others
        imgio(ref)
        return
    if sys.argv[1:] == ["ba"]:
        ba(ref)
        return
    if sys.argv[1:] == ["vs_ref"]:
        vs_ref(ref)
        return
    imgio(ref)
    ba(ref)
    vs_ref(ref)

    # ---- SIFT chain on one 240x180 view
    img = synth.make_canvas(180, 240, 101)
    tr = ref.sift_trace(img)
    pts = [tr.points(s) for s in range(3)]
    coor, desc = tr.descriptors()
    planes = {f"gauss_o{o}_l{l}_crc": plane_crc(tr.plane(1, o, l)) for o in range(4) for l in range(7)}
    planes.update({f"dog_o{o}_l{l}_crc": plane_crc(tr.plane(2, o, l)) for o in range(4) for l in range(6)})
    np.savez_compressed(OUT / "sift_240x180.npz", input_sha=np.array(sha(img)),
                        working_size=np.array(tr.working_size()),
                        octave_sizes=np.array([tr.octave_size(o) for o in range(4)]),
                        dog_o0_l3=tr.plane(2, 0, 3)[40:60, 50:90].copy(),
                        raw=pts[0], refined=pts[1], oriented=pts[2], coor=coor, desc=desc, **planes)
    print("sift:", [len(p) for p in pts], desc.shape)

    # ---- matcher: two overlapping views + a noisy synthetic pair near the ratio threshold
    imgs, org = synth.make_stack(2, 240, 180, 90, 102)
    d0 = ref.sift_detect(imgs[0])[1]
    d1 = ref.sift_detect(imgs[1])[1]
    rng = np.random.RandomState(5)
    a = synth.rootsift_like(300, 6)
    b = (a[rng.permutation(300)][:260] + rng.randn(260, 128).astype(np.float32) * 28.0).astype(np.float32)
    c = (a[rng.permutation(300)][:280] + rng.randn(280, 128).astype(np.float32) * 38.0).astype(np.float32)
    np.savez_compressed(OUT / "match.npz", input_sha=np.array(sha(imgs[0], imgs[1], a, b, c)), d0=d0, d1=d1,
                        pairs_01=ref.match(d0, d1), pairs_10=ref.match(d1, d0), a=a, b=b, c=c,
                        pairs_ab=ref.match(a, b), pairs_ba=ref.match(b, a),
                        pairs_ac=ref.match(a, c), pairs_ca=ref.match(c, a))
    print("near-threshold pair:", len(ref.match(a, c)), "of 280")
    print("match:", len(d0), len(d1), len(ref.match(d0, d1)), len(ref.match(a, b)))

    # ---- cylinder warp
    wimg = synth.make_canvas(80, 120, 103)
    k = np.array([[10.5, -20.25], [-40.0, 30.0], [0.0, 0.0]])
    out, kk = ref.cyl_warp(wimg, k, 1.0)
    out2, kk2 = ref.cyl_warp(wimg, k, 0.9)
    np.savez_compressed(OUT / "cyl_warp_120x80.npz", input_sha=np.array(sha(wimg)),
                        shape=np.array(ref.cyl_warp_shape(120, 80)),
                        out=out, kpts_in=k, kpts_out=kk, out_h09=out2, kpts_out_h09=kk2)
    print("warp:", out.shape)

    # ---- blenders on 3 views of 120x80
    bimgs, borg = synth.make_stack(3, 120, 80, 40, 104)
    items, geom = synth.translation_blend_setup(borg, 120, 80)
    res = {}
    for lazy in (0, 1):
        for ordered in (0, 1):
            res[f"linear_lazy{lazy}_ord{ordered}"] = ref.blend(bimgs, items, geom, 0,
                                                               default_params(lazy_read=lazy, ordered_input=ordered))
    for bands in (1, 3, 5):
        res[f"multiband_{bands}"] = ref.blend(bimgs, items, geom, bands)
    np.savez_compressed(OUT / "blend_3x120x80.npz", input_sha=np.array(sha(*bimgs)), **res)
    print("blend:", {k: v.shape for k, v in res.items()})


if __name__ == "__main__":
    main()
