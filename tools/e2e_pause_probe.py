#!/usr/bin/env python
"""Where do the 0.1 - 2 s pauses between e2e job completions come from?

Runs the bench's e2e leg (StitchLanes, 3 lanes, rgb8 boundary) for N jobs with every
engine call of every lane timed, next to two heartbeats:
  * host heartbeat: a thread that sleeps 1 ms in a loop — a gap there means the whole
    process (or the CPU it runs on) stalled;
  * GPU heartbeat: a second context that records + waits one event per ms on its own
    stream — a gap there and not in the host heartbeat means the driver / GPU stalled.
Prints the slowest calls and the heartbeat gaps that overlap them.

  python tools/e2e_pause_probe.py [jobs=600]
"""
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from openpano_b200.stitcher import StitchLanes  # noqa: E402

n_jobs = int(sys.argv[1]) if len(sys.argv) > 1 else 600
torch.cuda.set_device(0)
bench.bind_to_gpu_numa_node(0)
imgs, pairs, items, geom, params, mpx, pix = bench.make_workload(0, 0)
shapes = [im.shape[:2] for im in imgs]
out_w, out_h = max(it[2] for it in items), max(it[3] for it in items)

lanes = StitchLanes(0, params, lanes=3, depth=2, rgb8=True, crop=True)
src = [torch.from_numpy(p).pin_memory() for p in pix]
outs = [torch.empty(lanes.out_bytes((out_w, out_h)), dtype=torch.uint8).pin_memory() for _ in range(9)]
ptrs = [t.data_ptr() for t in src]


def jobs(n):
    return [(ptrs, shapes, (out_w, out_h), pairs, items, geom, outs[i % 9].data_ptr(), 0) for i in range(n)]


calls = []          # (t0, t1, lane, name)
marks = []          # (lane, name, host time, torch event) — GPU-side timeline of every job
ref_ev = torch.cuda.Event(enable_timing=True)
ref_ev.record()
torch.cuda.synchronize()
t_ref = time.perf_counter()


def wrap(obj, name, lane, label, before=None, after=None):
    fn = getattr(obj, name)

    def wrapped(*a, **k):
        if before:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(before[1])
            marks.append((lane, before[0], time.perf_counter(), ev))
        t0 = time.perf_counter()
        r = fn(*a, **k)
        t1 = time.perf_counter()
        calls.append((t0, t1, lane, label))
        if after:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(after[1])
            marks.append((lane, after[0], t1, ev))
        return r
    setattr(obj, name, wrapped)


for q, ps in enumerate(lanes.lanes):
    s_up, s_cmp, s_dn = (torch.cuda.ExternalStream(e.stream) for e in (ps.up, ps.cmp, ps.dn))
    wrap(ps.cmp, "sift_detect_batch_rgb8_ptr", q, "cmp.sift", before=("c0 compute starts", s_cmp),
         after=("c1 sift enqueued", s_cmp))
    wrap(ps.cmp, "match_pairs", q, "cmp.match_pairs", after=("c2 match lists on host", s_cmp))
    wrap(ps.cmp, "blend_rgb8_dev", q, "cmp.blend")
    wrap(ps.cmp, "event_record", q, "cmp.event_record", before=("c3 blend+convert enqueued", s_cmp))
    wrap(ps.dn, "dev_download_async", q, "dn.download_async", after=("d1 download enqueued", s_dn))
    wrap(ps.cmp, "event_wait", q, "cmp.event_wait")
    wrap(ps, "stage", q, "stage", before=("u0 stage starts", s_up), after=("u1 uploads enqueued", s_up))
    wrap(ps, "run", q, "run")
    wrap(ps, "wait", q, "wait")

stop = False
host_beats, gpu_beats = [], []


def host_heartbeat():
    while not stop:
        host_beats.append(time.perf_counter())
        time.sleep(0.001)


def gpu_heartbeat():
    s = torch.cuda.Stream()
    ev = torch.cuda.Event()
    while not stop:
        ev.record(s)
        ev.synchronize()
        gpu_beats.append(time.perf_counter())
        time.sleep(0.001)


lanes.map(jobs(18))
torch.cuda.synchronize()
th = [threading.Thread(target=host_heartbeat, daemon=True), threading.Thread(target=gpu_heartbeat, daemon=True)]
for t in th:
    t.start()
calls.clear()
t_start = time.perf_counter()
lanes.map(jobs(n_jobs))
torch.cuda.synchronize()
t_end = time.perf_counter()
stop = True
for t in th:
    t.join()

done = np.sort(np.array(lanes.done_times))
gaps = np.diff(np.concatenate([[t_start], done]))
print(f"{n_jobs} jobs in {t_end - t_start:.3f} s = {(t_end - t_start) / n_jobs * 1e3:.3f} ms/job; "
      f"median gap {np.median(gaps) * 1e3:.2f} ms, gaps > 20 ms: {(gaps > 0.02).sum()}, sum {gaps[gaps > 0.02].sum():.3f} s")


def beat_gaps(beats, lo, hi):
    b = np.array([x for x in beats if lo - 0.05 <= x <= hi + 0.05])
    return float(np.diff(b).max() * 1e3) if len(b) > 1 else float("nan")


hb, gb = np.diff(np.array(host_beats)), np.diff(np.array(gpu_beats))
print(f"host heartbeat: {len(host_beats)} beats, max gap {hb.max() * 1e3:.1f} ms, gaps > 10 ms: {(hb > 0.01).sum()}")
print(f"gpu  heartbeat: {len(gpu_beats)} beats, max gap {gb.max() * 1e3:.1f} ms, gaps > 10 ms: {(gb > 0.01).sum()}")
runs = sorted([c for c in calls if c[3] == "run"], key=lambda c: c[0] - c[1])[:6]
print("slowest run() calls (ms, lane, at s | host-heartbeat / gpu-heartbeat max gap around it), their sub-calls, and")
print("the GPU-side marks recorded during them (host time s -> time the stream reached the mark, s):")
for t0, t1, q, name in runs:
    print(f"  {(t1 - t0) * 1e3:8.1f}  lane {q}  run  at {t0 - t_start:7.3f}  | {beat_gaps(host_beats, t0, t1):7.1f} / {beat_gaps(gpu_beats, t0, t1):7.1f}")
    for c in calls:
        if c[2] == q and c[3] not in ("run",) and t0 <= c[0] and c[1] <= t1 and c[1] - c[0] > 0.002:
            print(f"        sub-call {c[3]:22s} {(c[1] - c[0]) * 1e3:8.1f} ms at {c[0] - t_start:7.3f}")
    for (lq, label, th, ev) in marks:
        if lq == q and t0 - 0.01 <= th <= t1 + 0.01:
            print(f"        mark {label:28s} host {th - t_start:7.3f}  gpu {(t_ref - t_start) + ref_ev.elapsed_time(ev) / 1e3:7.3f}")
by = {}
for t0, t1, q, name in calls:
    by.setdefault(name, []).append(t1 - t0)
for name, v in by.items():
    v = np.array(v) * 1e3
    print(f"  {name:5s}: n {len(v)}, median {np.median(v):.3f} ms, p99 {np.percentile(v, 99):.3f}, max {v.max():.1f}")
lanes.close()
