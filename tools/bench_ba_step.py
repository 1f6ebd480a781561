#!/usr/bin/env python
"""Per-LM-iteration cost of bundle adjustment's per-point work (incremental_bundle_adjuster.cc:117-169) on
the device session against today's path, for the 38-camera case and the >= 600 k-row case of
tests/test_gpu_ba.py.  One JSON line per case:

  session        pano_ba_error + pano_ba_normal_equations (J, J^T J, b), no residual download: host wall
                 time per call (every call ends in a host wait) and, in a separate profiled pass, the
                 device time of each kernel (k_ba_error_sum on its own among them)
  today          pano_ba_jacobian(want_rows) + calcError on the host (the oracle's C restatement of the
                 reference loop, -O2) + J^T r on the host over the downloaded compact rows (numpy)
  pcie_bytes     both paths per iteration, computed from shapes (not measured)
  device         card name, power limit and max SM clock, read in the same run

    python tools/bench_ba_step.py [--iters 20] [--warmup 3] [--out results/bench_ba_step.jsonl]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from openpano_b200.capi import Engine  # noqa: E402
from tests import ba_step_util as bs  # noqa: E402
from tests.ba_util import ba_case, numpy_pair_mats  # noqa: E402
from tests.checker import get_checker  # noqa: E402

CASES = [(38, 400, 7, 60), (24, 9000, 8, 16)]
PAIR_TABLE_B = 4 * 4 + 13 * 9 * 8          # pano_ba_pair


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": "not available", "error": str(e)}


def pcie_bytes(n_cam, n_pair, nm):
    n = 6 * n_cam
    jtj, b = n * n * 8, n * 8
    return {
        "session_up": n_pair * 72 + n_pair * PAIR_TABLE_B,          # Hto_to_from, then the pair table with the 13 matrices
        "session_down": jtj + b + 16,                                # J^T J, b, avg, max
        "today_up": n_pair * PAIR_TABLE_B + nm * 16,                 # pair table + p.first of every match
        "today_down": nm * 24 * 8 + jtj,                             # compact J rows + J^T J
    }


def host_jtr(n_cam, pairs, rows, res):
    """J^T r over the compact rows (sparse; a different summation order from the reference's, timing only)."""
    nm = len(rows)
    prod = rows[:, :12] * res[0::2, None] + rows[:, 12:] * res[1::2, None]
    cols = np.empty((nm, 12), np.int64)
    begin = 0
    for f, t, k in pairs:
        cols[begin:begin + k, :6] = 6 * f + np.arange(6)
        cols[begin:begin + k, 6:] = 6 * t + np.arange(6)
        begin += k
    return np.bincount(cols.ravel(), prod.ravel(), minlength=6 * n_cam)


def run_case(eng, orc, args, iters, warmup):
    n_cam, per_pair, seed, extra = args
    cams, pairs, pts = ba_case(n_cam, per_pair, seed, extra_pairs=extra)
    mats = numpy_pair_mats(cams, pairs)
    htos = [mats[:, 0], numpy_pair_mats(bs.rejected_cams(cams, 1), pairs)[:, 0]]
    nm = len(pts)
    jpairs = [(f, t, k, m) for (f, t, k), m in zip(pairs, mats)]

    s = eng.ba_session(n_cam, pairs, pts)
    try:
        def lm_iteration(i):
            t0 = time.perf_counter()
            s.error(htos[i & 1], want_residuals=False)
            t1 = time.perf_counter()
            s.normal_equations(mats)
            t2 = time.perf_counter()
            return t1 - t0, t2 - t1

        for i in range(warmup):
            lm_iteration(i)
        wall = np.array([lm_iteration(i) for i in range(iters)]) * 1e3
        # device time per kernel, in a pass of its own with the event profiler on
        eng.profile(True)
        eng.profile_reset()
        for i in range(iters):
            lm_iteration(i)
        prof = eng.profile_read()
        eng.profile(False)
    finally:
        s.close()
    kernels = {k: round(v[1] / iters, 4) for k, v in prof.items()}
    err_kernels = ("k_ba_residuals", "k_ba_error_sum")
    ne_kernels = ("k_ba_rows", "k_ba_jtj", "k_ba_jtr")

    # today's path: pano_ba_jacobian(want_rows) + host calcError + host J^T r over the downloaded rows
    def today():
        t0 = time.perf_counter()
        rows, _ = eng.ba_jacobian(n_cam, jpairs, pts[:, :2], want_rows=True)
        t1 = time.perf_counter()
        res, _, _ = bs.orc_error(pairs, htos[0], pts)
        t2 = time.perf_counter()
        host_jtr(n_cam, pairs, rows, res)
        t3 = time.perf_counter()
        return t1 - t0, t2 - t1, t3 - t2

    for _ in range(warmup):
        today()
    tw = np.array([today() for _ in range(iters)]) * 1e3
    return {
        "case": {"n_cam": n_cam, "pairs": len(pairs), "matches": nm, "j_rows": 2 * nm},
        "session_ms": {"ba_error_wall": round(float(np.median(wall[:, 0])), 4),
                       "normal_equations_wall": round(float(np.median(wall[:, 1])), 4),
                       "iteration_wall": round(float(np.median(wall.sum(1))), 4),
                       "ba_error_kernels": round(sum(kernels.get(k, 0.0) for k in err_kernels), 4),
                       "normal_equations_kernels": round(sum(kernels.get(k, 0.0) for k in ne_kernels), 4),
                       "k_ba_error_sum": kernels.get("k_ba_error_sum"),
                       "per_kernel": kernels},
        "today_ms": {"ba_jacobian_with_rows_wall": round(float(np.median(tw[:, 0])), 4),
                     "host_calc_error": round(float(np.median(tw[:, 1])), 4),
                     "host_jtr_numpy": round(float(np.median(tw[:, 2])), 4),
                     "iteration_wall": round(float(np.median(tw.sum(1))), 4)},
        "pcie_bytes_per_iteration": pcie_bytes(n_cam, len(pairs), nm),
        "iters": iters,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = device_info()
    eng = Engine(0)
    orc = get_checker("orc")
    lines = []
    for args in CASES:
        r = run_case(eng, orc, args, a.iters, a.warmup)
        r["device"] = dev
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    eng.close()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
