#!/usr/bin/env python
"""Multi-GPU check of the sharded hot path (SURVEY.md §8e) — launch with torchrun:

  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 \
      tools/run_dist.py [small|unordered38] [reps] [bands] [rgb8] [gauss_window_factor=N]

Every rank SIFTs its images (k mod G), descriptors are all-gathered over NCCL, pair
tasks are dealt, strips of the mosaic are blended per rank and gathered.  Rank 0 then
repeats the whole job on its own GPU alone and checks that the match lists and the
mosaic are bit-identical, and prints one JSON line with per-phase device times.

rgb8: the stack is quantised to 8-bit pixels (image 1 as a grey H×W image among colour ones) and run
through DistributedStitcher.run_rgb8; the one-GPU job reads the same pixels (SIFT from 8-bit pixels +
pano_blend_rgb8_dev).  gauss_window_factor=N: the composite's GAUSS_WINDOW_FACTOR (e.g. 12 with 16
bands: a multiband strip halo of 288 rows)."""
import json
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from openpano_b200 import synth  # noqa: E402
from openpano_b200._abi import default_params  # noqa: E402
from openpano_b200.capi import Engine  # noqa: E402
from openpano_b200.parallel import DistributedStitcher, shard_images  # noqa: E402
from openpano_b200.stitcher import all_pairs  # noqa: E402


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "small"
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    bands = int(sys.argv[3]) if len(sys.argv) > 3 else 0
    rgb8 = "rgb8" in sys.argv[4:]
    bparams = default_params()
    for arg in sys.argv[4:]:
        if arg.startswith("gauss_window_factor="):
            bparams.gauss_window_factor = int(arg.split("=", 1)[1])
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    if which == "small":
        imgs, org = synth.make_stack(7, 320, 240, 110, 31, rows=2, step_y=80)
        name = "7x320x240, all pairs"
    else:
        imgs, org = synth.config_stack("unordered_38x1300x867")
        name = "config 3: 38x1300x867 unordered, all pairs"
    n = len(imgs)
    h, w = imgs[0].shape[:2]
    items, geom = synth.translation_blend_setup(org, w, h)
    pairs = all_pairs(n)
    shapes = [im.shape[:2] for im in imgs]
    params = default_params()
    pix = None
    if rgb8:
        pix = [(im * 255.0 + 0.5).astype(np.uint8) for im in imgs]
        pix[1] = np.ascontiguousarray(pix[1][..., 1])
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng = Engine(local, stream.cuda_stream)
        src = pix if rgb8 else imgs
        owned = {k: torch.from_numpy(src[k]).to("cuda", non_blocking=False) for k in shard_images(n, world, rank)}
        ds = DistributedStitcher(eng, params, bparams)
        best = None
        for rep in range(reps):
            torch.cuda.synchronize()
            dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run = ds.run_rgb8 if rgb8 else ds.run
            matches, mosaic = run(owned, n, shapes, pairs, items, geom, bands)
            e1.record()
            torch.cuda.synchronize()
            t = torch.tensor([e0.elapsed_time(e1)], device="cuda")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            if best is None or t.item() < best[0]:
                best = (t.item(), dict(ds.ms), dict(ds.host_ms))
        res = None
        if rank == 0:
            # the same job on this GPU alone
            all_dev = [torch.from_numpy(im).cuda() for im in src]
            ptrs = [t_.data_ptr() for t_ in all_dev]
            ws, hs = [s[1] for s in shapes], [s[0] for s in shapes]
            chans = [1 if im.ndim == 2 else 3 for im in src]
            torch.cuda.synchronize()
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for rep in range(2):
                s0.record()
                if rgb8:
                    fs = eng.sift_detect_batch_rgb8_ptr(ptrs, ws, hs, chans, params, device=True)
                else:
                    fs = eng.sift_detect_batch_ptr(ptrs, ws, hs, params, device=True)
                ref_m = eng.match_pairs(fs, pairs, params)
                tw, th = max(it[2] for it in items), max(it[3] for it in items)
                ref_out = torch.empty((th, tw, 3), dtype=torch.float32, device="cuda")
                if rgb8:
                    eng.blend_rgb8_dev(ptrs, chans, shapes, items, geom, ref_out.data_ptr(), tw, th, bands, bparams)
                else:
                    eng.blend_dev(ptrs, shapes, items, geom, ref_out.data_ptr(), tw, th, bands, bparams)
                s1.record()
                torch.cuda.synchronize()
                fs.free()
            same_m = all(np.array_equal(a, b) for a, b in zip(matches, ref_m)) and len(matches) == len(ref_m)
            same_o = bool(torch.equal(mosaic, ref_out))
            mpx = sum(s[0] * s[1] for s in shapes) / 1e6
            res = {"workload": name, "bands": bands, "rgb8": rgb8, "gauss_window_factor": bparams.gauss_window_factor, "n_gpus": world, "images": n, "pairs": len(pairs), "ms_sharded": round(best[0], 3),
                   "phase_ms_rank0": {k: round(v, 3) for k, v in best[1].items()},
                   "phase_host_ms_rank0": {k: round(v, 3) for k, v in best[2].items()},
                   "ms_one_gpu": round(s0.elapsed_time(s1), 3), "mpx_per_s_sharded": round(mpx / best[0] * 1e3, 1),
                   "matches": int(sum(len(m) for m in matches)), "matches_identical": bool(same_m),
                   "mosaic_identical": same_o}
            print(json.dumps(res), flush=True)
        eng.close()
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0 and not (res["matches_identical"] and res["mosaic_identical"]):
        sys.exit(1)


if __name__ == "__main__":
    main()
