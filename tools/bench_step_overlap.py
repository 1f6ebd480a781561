"""bench.py's `value` step with the library build and the call order of the step chosen independently: the 2×2 of
old / new library × old / new order, alternated, and optionally a torch.profiler timeline of a few steps.

  python tools/bench_step_overlap.py --old openpano_b200/_variants/parent.so [--new LIB] [--orders old,new]
                                     [--reps 6] [--steps 100] [--trace DIR]

Orders:
  old   the composite is enqueued on the second context first, then SIFT and the matcher
  new   Stitcher.run_device as it ships (order b)
  a     SIFT first; the composite waits for the images only
  b     SIFT first; the composite waits for an event recorded after SIFT's last kernel
  c     the composite is queued once the match result is on the host
Each arm (library × order) runs in a worker process of its own (PANO_B200_LIB names the library).  Every
repetition times `--steps` steps of each arm the way bench.py's value loop does (CUDA events around the
steps, collector off), the arms' order reversed every repetition.  Each arm reports the median ms per step
of the repetitions, with the spread (min, max) and every value.  `same` says every arm gave the same bytes
for the features, the match total and the mosaic.

--trace DIR writes a torch.profiler trace of 6 steps per arm (DIR/<arm>.json) and prints per step:
  idle_ms         GPU time with no kernel running, from the step's first kernel to the next step's first
  to_sift_ms      host start of the step to the start of SIFT's first kernel
  blend           start and end of k_linear_blend, SIFT's first kernel start, k_descriptor's end and the step's
                  last kernel end, all in ms from the step's first kernel
  sift_call_ms    host time of the sift_detect_batch_ptr call
The card's name and power limit are read in the same run.  Needs an H100."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

SIFT_KERNELS = ("k_pyramid_grey", "k_blur_extrema", "k_extrema_seams", "k_rank_sort", "k_refine", "k_orientation",
                "k_expand_scan", "k_descriptor", "k_blur_dog", "k_extrema_scan")
TRACE_STEPS = 6


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


# ----------------------------------------------------------------------------- step orders
def _sift(st):
    shapes = st._shapes
    return st.eng.sift_detect_batch_ptr(st.image_ptrs(), [s[1] for s in shapes], [s[0] for s in shapes], st.params,
                                        device=True)


def _blend(st, items, geom, bands):
    aux = st._aux_engine()
    aux.event_wait(st._ev_in)
    aux.blend_dev(st.image_ptrs(), st._shapes, items, geom, st._d_out, st._out_shape[0], st._out_shape[1], bands,
                  st.params)
    aux.event_record(st._ev_blend)


def _finish(st, fs, pairs):
    total = st.eng.match_pairs_dev(fs, pairs, st.params)
    st.eng.event_wait(st._ev_blend)
    return fs, total


def step_old(st, pairs, items, geom, bands):
    st._aux_engine()
    st.eng.event_record(st._ev_in)
    _blend(st, items, geom, bands)
    return _finish(st, _sift(st), pairs)


def step_a(st, pairs, items, geom, bands):
    st._aux_engine()
    st.eng.event_record(st._ev_in)
    fs = _sift(st)
    _blend(st, items, geom, bands)
    return _finish(st, fs, pairs)


def step_b(st, pairs, items, geom, bands):
    st._aux_engine()
    fs = _sift(st)
    st.eng.event_record(st._ev_in)
    _blend(st, items, geom, bands)
    return _finish(st, fs, pairs)


def step_c(st, pairs, items, geom, bands):
    st._aux_engine()
    fs = _sift(st)
    total = st.eng.match_pairs_dev(fs, pairs, st.params)
    st.eng.event_record(st._ev_in)
    _blend(st, items, geom, bands)
    st.eng.event_wait(st._ev_blend)
    return fs, total


def step_new(st, pairs, items, geom, bands):
    return st.run_device(pairs, items, geom, bands, want_matches=False)


ORDERS = {"old": step_old, "new": step_new, "a": step_a, "b": step_b, "c": step_c}


# ----------------------------------------------------------------------------- timeline
def timeline(path, n_steps):
    """Per-step figures from a chrome trace written by torch.profiler (see the module docstring)."""
    ev = json.loads(Path(path).read_text())["traceEvents"]
    steps = sorted((e for e in ev if e.get("cat") == "user_annotation" and e.get("name") == "overlap_step"), key=lambda e: e["ts"])
    calls = sorted((e for e in ev if e.get("cat") == "user_annotation" and e.get("name") == "sift_detect_batch_ptr"),
                   key=lambda e: e["ts"])
    launch_ts = {e["args"]["correlation"]: e["ts"] for e in ev
                 if e.get("ph") == "X" and e.get("cat") in ("cuda_runtime", "cuda_driver")
                 and "correlation" in e.get("args", {})}
    kernels = [e for e in ev if e.get("ph") == "X" and e.get("cat") == "kernel"]
    per = [[] for _ in steps]
    for k in kernels:
        # a kernel belongs to the step whose host range launched it; without launch records, to the last step
        # that started before it
        t = launch_ts.get(k["args"].get("correlation"))
        if t is None:
            t = max((s["ts"] for s in steps if s["ts"] <= k["ts"]), default=None)
            if t is None:
                continue
        for i, s in enumerate(steps):
            if s["ts"] <= t <= s["ts"] + s["dur"]:
                per[i].append(k)
                break
    out = []
    for i in range(len(steps) - 1):
        ks = sorted(per[i], key=lambda k: k["ts"])
        nxt = min(k["ts"] for k in per[i + 1]) if per[i + 1] else None
        if not ks or nxt is None:
            continue
        t0 = ks[0]["ts"]
        busy, cur_s, cur_e = 0.0, None, None
        for k in sorted(per[i] + per[i + 1], key=lambda k: k["ts"]):
            s, e = max(k["ts"], t0), min(k["ts"] + k["dur"], nxt)
            if e <= s:
                continue
            if cur_e is None or s > cur_e:
                busy += (cur_e - cur_s) if cur_e is not None else 0.0
                cur_s, cur_e = s, e
            else:
                cur_e = max(cur_e, e)
        busy += (cur_e - cur_s) if cur_e is not None else 0.0
        sift = [k for k in ks if any(n in k["name"] for n in SIFT_KERNELS)]
        blend = [k for k in ks if "k_linear_blend" in k["name"]]
        desc = [k for k in ks if "k_descriptor" in k["name"]]
        rel = lambda t: round((t - t0) / 1e3, 4)  # noqa: E731
        row = dict(step=i, idle_ms=round((nxt - t0 - busy) / 1e3, 4),
                   to_sift_ms=round((sift[0]["ts"] - steps[i]["ts"]) / 1e3, 4) if sift else None,
                   sift_start=rel(sift[0]["ts"]) if sift else None,
                   sift_end=rel(desc[-1]["ts"] + desc[-1]["dur"]) if desc else None,
                   blend_start=rel(blend[0]["ts"]) if blend else None,
                   blend_end=rel(blend[-1]["ts"] + blend[-1]["dur"]) if blend else None,
                   step_end=rel(max(k["ts"] + k["dur"] for k in ks)),
                   sift_call_ms=round(calls[i]["dur"] / 1e3, 4) if i < len(calls) else None)
        out.append(row)
    return out[:n_steps]


# ----------------------------------------------------------------------------- worker (one arm)
def worker(order):
    out = os.fdopen(os.dup(1), "w")     # replies only; anything else the process prints goes to stderr
    os.dup2(2, 1)
    import gc
    import torch
    import bench
    from openpano_b200.capi import Engine
    from openpano_b200.stitcher import Stitcher

    imgs, pairs, items, geom, params, _, _ = bench.make_workload(0, 0)
    shapes = [im.shape[:2] for im in imgs]
    out_w, out_h = max(it[2] for it in items), max(it[3] for it in items)
    stream = torch.cuda.Stream()
    step_fn = ORDERS[order]
    with torch.cuda.stream(stream):
        eng = Engine(0, stream.cuda_stream)
        st = Stitcher(eng, params)
        host = [torch.from_numpy(im).pin_memory() for im in imgs]
        st.upload([t.data_ptr() for t in host], shapes, (out_w, out_h))
        eng.sync()
        sift_call = eng.sift_detect_batch_ptr

        def step():
            fs, total = step_fn(st, pairs, items, geom, 0)
            return fs, total

        def steps(k):
            for _ in range(k):
                step()[0].free()

        gc.collect()
        gc.disable()
        steps(5)
        torch.cuda.synchronize()
        for line in sys.stdin:
            cmd = json.loads(line)
            op = cmd["cmd"]
            if op == "time":
                l0 = eng.launch_count()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                steps(cmd["steps"])
                e1.record(stream)
                torch.cuda.synchronize()
                reply = {"ms": e0.elapsed_time(e1) / cmd["steps"], "launches": (eng.launch_count() - l0) / cmd["steps"]}
            elif op == "digest":
                fs, total = step()
                torch.cuda.synchronize()
                h = hashlib.sha256()
                for i in range(len(imgs)):
                    c, d = fs.download(i)
                    h.update(c.tobytes())
                    h.update(d.tobytes())
                fs.free()
                h.update(str(total).encode())
                mosaic = torch.empty((out_h, out_w, 3), dtype=torch.float32)
                eng.dev_download(mosaic.numpy(), st._d_out)
                h.update(mosaic.numpy().tobytes())
                reply = {"sha256": h.hexdigest()}
            elif op == "trace":
                from torch.profiler import ProfilerActivity, profile, record_function

                def timed_sift(*a, **k):
                    with record_function("sift_detect_batch_ptr"):
                        return sift_call(*a, **k)

                eng.sift_detect_batch_ptr = timed_sift
                with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    for _ in range(TRACE_STEPS + 1):
                        with record_function("overlap_step"):
                            fs, _ = step()
                        fs.free()
                    torch.cuda.synchronize()
                eng.sift_detect_batch_ptr = sift_call
                prof.export_chrome_trace(cmd["path"])
                reply = {"steps": timeline(cmd["path"], TRACE_STEPS)}
            else:
                break
            print(json.dumps(reply), file=out, flush=True)
        st.close()
        eng.close()


class Worker:
    def __init__(self, lib, order):
        env = dict(os.environ)
        if lib:
            env["PANO_B200_LIB"] = str(Path(lib).resolve())
        else:
            env.pop("PANO_B200_LIB", None)
        self.p = subprocess.Popen([sys.executable, __file__, "--worker", order], stdin=subprocess.PIPE,
                                  stdout=subprocess.PIPE, text=True, env=env, cwd=str(ROOT))

    def call(self, **cmd):
        self.p.stdin.write(json.dumps(cmd) + "\n")
        self.p.stdin.flush()
        line = self.p.stdout.readline()
        if not line:
            raise SystemExit(f"worker exited with {self.p.wait()}")
        return json.loads(line)

    def close(self):
        self.p.stdin.write(json.dumps({"cmd": "quit"}) + "\n")
        self.p.stdin.close()
        self.p.wait()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old", help="library of the parent build (required)")
    ap.add_argument("--new", default=None, help="library of this build (default: the in-tree build)")
    ap.add_argument("--orders", default="old,new", help=f"comma list of {','.join(ORDERS)}")
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--trace", metavar="DIR", default=None)
    ap.add_argument("--worker", metavar="ORDER", default=None)
    a = ap.parse_args()
    if a.worker:
        worker(a.worker)
        return
    if not a.old:
        ap.error("--old is required")
    info = gpu_info()
    arms = {f"{lib}_lib/{order}_order": Worker(a.old if lib == "old" else a.new, order)
            for lib in ("old", "new") for order in a.orders.split(",")}
    names = list(arms)
    ms = {k: [] for k in names}
    launches = {}
    for r in range(a.reps):
        for k in (names if r % 2 == 0 else names[::-1]):
            rep = arms[k].call(cmd="time", steps=a.steps)
            ms[k].append(rep["ms"])
            launches[k] = rep["launches"]
    digests = {k: arms[k].call(cmd="digest")["sha256"] for k in names}
    rows = {k: dict(median_ms=round(statistics.median(v), 4), min_ms=round(min(v), 4), max_ms=round(max(v), 4),
                    all_ms=[round(x, 4) for x in v], launches_per_step=launches[k]) for k, v in ms.items()}
    traces = {}
    if a.trace:
        os.makedirs(a.trace, exist_ok=True)
        for k in names:
            traces[k] = arms[k].call(cmd="trace", path=os.path.join(a.trace, k.replace("/", "__") + ".json"))["steps"]
            for row in traces[k]:
                print(k, json.dumps(row), file=sys.stderr, flush=True)
    for w in arms.values():
        w.close()
    print(json.dumps(dict(**info, reps=a.reps, steps=a.steps, old=a.old, new=a.new or "in-tree",
                          same=len(set(digests.values())) == 1, arms=rows, traces=traces)))


if __name__ == "__main__":
    main()
