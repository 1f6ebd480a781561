"""Diagnostic: host-side timeline of PipelinedStitcher (rgb8 or mat32f boundary) and the
event-timed kernels of its compute context.

  python tools/diag_pipeline.py [rgb8|f32] [depth]
"""
import sys, time
sys.path.insert(0, '.')
import numpy as np, torch
import bench
from openpano_b200.stitcher import PipelinedStitcher

rgb8 = (sys.argv[1] if len(sys.argv) > 1 else "rgb8") == "rgb8"
depth = int(sys.argv[2]) if len(sys.argv) > 2 else 3
imgs, pairs, items, geom, params, mpx, pix = bench.make_workload(0, 0)
shapes = [im.shape[:2] for im in imgs]
ow, oh = max(it[2] for it in items), max(it[3] for it in items)
ps = PipelinedStitcher(0, params, depth=depth, rgb8=rgb8, crop=True)
host = [torch.from_numpy(a).pin_memory() for a in (pix if rgb8 else imgs)]
ptrs = [t.data_ptr() for t in host]
outs = [torch.empty(ps.out_bytes((ow, oh)), dtype=torch.uint8).pin_memory() for _ in range(3)]
T = time.perf_counter


def timed_run(k, out_ptr):
    s = ps.slots[k]; sh = s["shapes"]
    ws, hs = [q[1] for q in sh], [q[0] for q in sh]
    t0 = T(); ps.cmp.event_wait(s["ev_up"])
    if rgb8:
        p = [s["pix"] + o for o in s["pix_offs"]]
        fs = ps.cmp.sift_detect_batch_rgb8_ptr(p, ws, hs, [3] * len(sh), params, device=True)
    else:
        p = [s["imgs"] + o for o in s["offs"]]
        fs = ps.cmp.sift_detect_batch_ptr(p, ws, hs, params, device=True)
    t1 = T()
    m = ps.cmp.match_pairs(fs, pairs, params); t2 = T()
    ps.cmp.event_wait(s["ev_dn"])
    if rgb8:
        ps.cmp.blend_rgb8_dev(p, [3] * len(sh), sh, items, geom, s["out"], ow, oh, 0, params)
    else:
        ps.cmp.blend_dev(p, sh, items, geom, s["out"], ow, oh, 0, params)
    if rgb8:
        ps.cmp.crop_rect_dev(s["out"], ow, oh, s["out8"])
        ps.cmp.mat32f_to_rgb8_dev(s["out"], ow, oh, s["out8"], s["out8"] + ps.RGB8_HEADER)
    ps.cmp.event_record(s["ev_cmp"]); t3 = T()
    fs.free(); ps.dn.event_wait(s["ev_cmp"])
    ps.dn.dev_download_async(out_ptr, s["out8"] if rgb8 else s["out"], ps.out_bytes((ow, oh)))
    ps.dn.event_record(s["ev_dn"]); s["busy"] = True; t4 = T()
    return (k, m), (t1 - t0, t2 - t1, t3 - t2, t4 - t3)


N = 12
for trial in range(3):
    if trial == 2:
        ps.cmp.profile(True); ps.cmp.profile_reset()
    slot = ps.stage(ptrs, shapes, (ow, oh)); pending = None
    t_all = T()
    for i in range(N):
        a = T(); nxt = ps.stage(ptrs, shapes, (ow, oh)); b = T()
        job, parts = timed_run(slot, outs[i % 3].data_ptr()); c = T()
        if pending: ps.wait(pending)
        d = T()
        if trial == 1: print(f"i={i} stage {1e3*(b-a):6.2f}  run {1e3*(c-b):6.2f} [sift {1e3*parts[0]:5.2f} match {1e3*parts[1]:5.2f} blend {1e3*parts[2]:5.2f} dn {1e3*parts[3]:5.2f}] wait {1e3*(d-c):5.2f}")
        pending, slot = job, nxt
    ps.wait(pending)
    print("trial", trial, "avg per job ms", 1e3 * (T() - t_all) / N)
prof = ps.cmp.profile_read()
tot = 0
for name, (cnt, ms) in sorted(prof.items(), key=lambda kv: -kv[1][1]):
    print(f"{name:22s} {cnt / N:5.1f}/job {ms / N:8.4f} ms/job")
    tot += ms / N
print("kernel sum ms/job", tot)
ps.close()
