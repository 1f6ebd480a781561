"""Multi-GPU sharding of the hot path (SURVEY.md §8e): one process per GPU.

The reference is a single process whose parallel axes are independent units —
images in calc_feature (stitcherbase.cc:14), image pairs in pairwise_match
(stitcher.cc:106).  Across GPUs the same axes are sharded:

  SIFT           image k -> rank k mod G                       no collective
  exchange (C1)  every pair needs both descriptor sets         all-gather of
                 (matcher.cc:96-101)                            {count, desc, coor}
  matching       the task list of stitcher.cc:98-100 / :121-122 dealt by
                 descending N_i*N_j (longest-processing-time)   no collective
  results        match pairs are tiny                           gather to rank 0

Collectives go through torch.distributed (NCCL on GPUs, gloo in the CPU tests).
The compute is a *backend* object so that the same plumbing is exercised on CPU
(tests pass an oracle-backed backend) and on GPUs (EngineBackend below).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np


# ----------------------------------------------------------------------------- pure sharding logic
def shard_images(n_images: int, world: int, rank: int) -> List[int]:
    """Image k is owned by rank k mod world."""
    return [k for k in range(n_images) if k % world == rank]


def deal_pairs(pairs: Sequence[Tuple[int, int]], counts: Sequence[int], world: int) -> List[List[int]]:
    """Longest-processing-time assignment of pair tasks by cost N_i*N_j.
    Returns, per rank, the indices into `pairs` it matches (deterministic)."""
    order = sorted(range(len(pairs)), key=lambda t: (-counts[pairs[t][0]] * counts[pairs[t][1]], t))
    load = [0] * world
    out: List[List[int]] = [[] for _ in range(world)]
    for t in order:
        r = min(range(world), key=lambda q: (load[q], q))
        out[r].append(t)
        load[r] += counts[pairs[t][0]] * counts[pairs[t][1]] + 1
    for lst in out:
        lst.sort()
    return out


# ----------------------------------------------------------------------------- collectives
def _dist():
    import torch.distributed as dist
    return dist


def all_gather_features(local: dict, n_images: int, device=None):
    """C1: all-gather of the per-image descriptor blocks.

    local: {image index: (coor float64 [n,2], desc float32 [n,128])} owned by this
    rank.  Returns the full lists (coors, descs) for images 0..n_images-1 on every
    rank.  Variable sizes: counts first, then one padded all_gather."""
    import torch
    dist = _dist()
    world, rank = dist.get_world_size(), dist.get_rank()
    dev = device if device is not None else torch.device("cpu")
    counts = torch.zeros(n_images, dtype=torch.int64, device=dev)
    for k, (_, d) in local.items():
        counts[k] = len(d)
    dist.all_reduce(counts, op=dist.ReduceOp.SUM)
    counts_h = [int(c) for c in counts.cpu()]
    # per-rank payload: images it owns, concatenated in image order, padded to the largest rank payload
    owned = [shard_images(n_images, world, r) for r in range(world)]
    rows = [sum(counts_h[k] for k in owned[r]) for r in range(world)]
    pad = max(max(rows), 1)
    mine = torch.zeros((pad, 128 + 4), dtype=torch.float32, device=dev)   # 128 desc + 2 f64 coords as 4 f32 words
    off = 0
    for k in owned[rank]:
        c, d = local[k]
        n = len(d)
        if n:
            mine[off:off + n, :128] = torch.from_numpy(np.ascontiguousarray(d, np.float32)).to(dev)
            cw = torch.from_numpy(np.ascontiguousarray(c, np.float64).view(np.float32).reshape(n, 4)).to(dev)
            mine[off:off + n, 128:] = cw
        off += n
    gathered = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(gathered, mine)
    coors, descs = [None] * n_images, [None] * n_images
    for r in range(world):
        g = gathered[r].cpu().numpy()
        off = 0
        for k in owned[r]:
            n = counts_h[k]
            descs[k] = np.ascontiguousarray(g[off:off + n, :128])
            coors[k] = np.ascontiguousarray(g[off:off + n, 128:]).view(np.float64).reshape(n, 2)
            off += n
    return coors, descs


def gather_matches(my_tasks: Sequence[int], my_results: Sequence[np.ndarray], n_tasks: int):
    """Gather per-pair match arrays to rank 0 (returns the full list there, None elsewhere)."""
    dist = _dist()
    payload = [(int(t), np.ascontiguousarray(m, np.int32)) for t, m in zip(my_tasks, my_results)]
    out = [None] * dist.get_world_size() if dist.get_rank() == 0 else None
    dist.gather_object(payload, out, dst=0)
    if dist.get_rank() != 0:
        return None
    full = [None] * n_tasks
    for part in out:
        for t, m in part:
            full[t] = m
    return full


# ----------------------------------------------------------------------------- driver
def distributed_features_and_matches(backend, images: dict, n_images: int, pairs, device=None):
    """images: {image index: HxWx3 float32} for the images this rank owns
    (shard_images).  Every rank returns (coors, descs) for ALL images; rank 0 also
    gets the per-pair match arrays in task order (others get None)."""
    dist = _dist()
    world, rank = dist.get_world_size(), dist.get_rank()
    mine = sorted(images)
    assert mine == shard_images(n_images, world, rank), "images must follow shard_images()"
    feats = backend.detect([images[k] for k in mine])
    local = {k: f for k, f in zip(mine, feats)}
    coors, descs = all_gather_features(local, n_images, device)
    counts = [len(d) for d in descs]
    tasks = deal_pairs(pairs, counts, world)[rank]
    results = backend.match_pairs(descs, [pairs[t] for t in tasks])
    matches = gather_matches(tasks, results, len(pairs))
    return coors, descs, matches


class EngineBackend:
    """Compute backend on one GPU through the C ABI (openpano_b200.capi.Engine)."""

    def __init__(self, engine, params=None):
        from ._abi import default_params
        self.eng = engine
        self.params = params or default_params()

    def detect(self, imgs):
        if not imgs:
            return []
        fs = self.eng.sift_detect_batch(imgs, self.params)
        try:
            return [fs.download(i) for i in range(len(imgs))]
        finally:
            fs.free()

    def match_pairs(self, descs, pairs):
        if not pairs:
            return []
        used = sorted({i for p in pairs for i in p})
        remap = {k: q for q, k in enumerate(used)}
        fs = self.eng.featureset_upload([descs[k] for k in used])
        try:
            return self.eng.match_pairs(fs, [(remap[i], remap[j]) for i, j in pairs], self.params)
        finally:
            fs.free()


# ----------------------------------------------------------------------------- match lists on the wire
def pack_match_lists(results, ntask: int, out: np.ndarray) -> int:
    """One rank's share of the match lists as a flat int32 record: [number of matches per dealt task ...
    (ntask slots, unused ones 0), (i, j) (i, j) ...].  `out` must hold ntask + 2 * total ints; returns total."""
    tot = sum(len(m) for m in results)
    out[:ntask] = 0
    if len(results):
        out[:len(results)] = [len(m) for m in results]
        if tot:
            out[ntask:ntask + 2 * tot] = np.concatenate(results).reshape(-1)
    return tot


def unpack_match_lists(got: np.ndarray, dealt, ntask: int, pad: int, n_pairs: int):
    """The inverse over all ranks: `got` = the ranks' records, each padded to `pad` ints, concatenated in rank
    order; dealt[r] = the pair indices rank r decided, in the order of its record.  -> list of [c, 2] arrays."""
    full = [None] * n_pairs
    for r, mine in enumerate(dealt):
        nt = len(mine)
        if not nt:
            continue
        seg = got[r * pad:(r + 1) * pad]
        cuts = np.cumsum(seg[:nt].astype(np.int64))
        lists = np.split(seg[ntask:ntask + 2 * int(cuts[-1])].reshape(-1, 2).copy(), cuts[:-1])
        for t_, m in zip(mine, lists):
            full[t_] = m
    return full


# ----------------------------------------------------------------------------- device-resident path (NCCL)
class DistributedStitcher:
    """The sharded hot path with every payload resident in HBM (one instance per
    rank, `torch.distributed` initialised with the NCCL backend, the Engine created
    on torch's CURRENT non-default stream so engine kernels and NCCL order on it).

      SIFT      owned images (k mod G), read as they were passed: f32 (run) or
                8-bit pixels (run_rgb8)                             no collective
      C1        descriptors + coordinates: export_dev -> ncclAllGather -> import_dev
                (run_rgb8: each image's channel count travels with its count)
      match     the dealt pair tasks against the gathered featureset  no collective
      results   match lists -> every rank (one padded int32 all-gather, a few KB)
      images    every rank blends a strip of every image: ncclAllGather of the sources
                into slots of the largest H×W×3, issued on a side stream BEFORE SIFT
                so that it overlaps SIFT + C1 + matching.  run moves and holds 12 B/px
                of f32; run_rgb8 moves and holds 3 B/px of 8-bit pixels (a grey image
                fills a third of its slot) and makes no f32 copy of any source
      blend     rows [r·H/G, (r+1)·H/G) of the canvas (LinearBlender pixels are
                independent, blender.cc:37-96; MultiBandBlender strips are computed
                from ROIs clipped to the strip + the summed blur half-widths), read
                from the gathered sources as they are (pano_blend_rows_dev /
                pano_blend_rows_rgb8_dev)                           no collective
      C2        strips -> ncclAllGather -> the mosaic (bit-identical to one GPU)

    blend_params: the composite's parameters where they differ from detection and matching's (e.g. a
    GAUSS_WINDOW_FACTOR wider than the SIFT blur's 31 taps allow); defaults to params.
    """

    PHASES = ("sift", "exchange_descriptors", "match", "gather_matches", "exchange_images", "blend_strip", "gather_strips")

    def __init__(self, engine, params=None, blend_params=None):
        from ._abi import default_params
        self.eng = engine
        self.params = params or default_params()
        self.blend_params = blend_params or self.params
        self.ms = {}
        self.host_ms = {}         # host wall time spent inside each phase's calls (launch / sync overhead)
        self._side = None
        self._stage = {}

    def _pinned(self, key, n):
        """A pinned int32 staging buffer of at least n elements, kept across jobs (cudaHostAlloc is slow)."""
        import torch
        buf = self._stage.get(key)
        if buf is None or buf.numel() < n:
            buf = torch.empty(max(n, 1 << 16), dtype=torch.int32).pin_memory()
            self._stage[key] = buf
        return buf

    def _timed(self, name, fn):
        import time
        import torch
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        out = fn()
        e1.record()
        self.host_ms[name] = self.host_ms.get(name, 0.0) + (time.perf_counter() - t0) * 1e3
        self._events.append((name, e0, e1))
        return out

    def run(self, owned: dict, n_images: int, shapes, pairs, items, geom, bands: int = 0):
        """owned: {image index: cuda float32 tensor H×W×3} following shard_images().
        Returns (matches on rank 0 / None elsewhere, mosaic tensor th×tw×3 on every rank)."""
        return self._run(owned, None, n_images, shapes, pairs, items, geom, bands)

    def run_rgb8(self, owned_pix: dict, n_images: int, shapes, pairs, items, geom, bands: int = 0):
        """The same from decoded 8-bit pixels (what read_img starts from, imgio.cc:72): owned_pix =
        {image index: contiguous cuda uint8 tensor H×W (grey) or H×W×3}.  SIFT and the strip read the
        pixels themselves and convert every tap as read_img would (bit-identical to run on read_img's
        f32 images); the image exchange moves 3 B/px instead of 12, and no f32 copy of a source is made."""
        return self._run(None, owned_pix, n_images, shapes, pairs, items, geom, bands)

    def _run(self, owned, owned_pix, n_images, shapes, pairs, items, geom, bands):
        import torch
        dist = _dist()
        eng, params = self.eng, self.params
        world, rank = dist.get_world_size(), dist.get_rank()
        dev = torch.device("cuda", torch.cuda.current_device())
        owners = [shard_images(n_images, world, r) for r in range(world)]
        mine = owners[rank]
        rgb8 = owned_pix is not None
        assert sorted(owned_pix if rgb8 else owned) == mine, "images must follow shard_images()"
        own_ch = {}
        if rgb8:
            for k in mine:
                x = owned_pix[k]
                if (x.dtype != torch.uint8 or not x.is_contiguous() or tuple(x.shape[:2]) != tuple(shapes[k])
                        or not (x.dim() == 2 or (x.dim() == 3 and x.shape[2] in (1, 3)))):
                    raise ValueError(f"run_rgb8: image {k} must be a contiguous H×W or H×W×{{1,3}} uint8 tensor of "
                                     f"shape {tuple(shapes[k])}, got {x.dtype} {tuple(x.shape)}")
                own_ch[k] = 1 if x.dim() == 2 else int(x.shape[2])
        self._events = []
        self.host_ms = {}
        main = torch.cuda.current_stream()
        if self._side is None:
            self._side = torch.cuda.Stream()
        side = self._side

        # ---- inputs of the blend: every image on every rank.  Depends on the inputs only, so it is
        # queued first on a side stream and runs under SIFT / C1 / matching.
        max_el = max(h * w * 3 for (h, w) in shapes)
        per_rank = max(len(o) for o in owners)
        src = owned_pix if rgb8 else owned
        dt = torch.uint8 if rgb8 else torch.float32
        side.wait_stream(main)
        with torch.cuda.stream(side):
            ev_i0 = torch.cuda.Event(enable_timing=True)
            ev_i1 = torch.cuda.Event(enable_timing=True)
            ev_i0.record()
            my_i = torch.zeros((per_rank, max_el), dtype=dt, device=dev)
            for q, k in enumerate(mine):
                my_i[q, :src[k].numel()] = src[k].reshape(-1)
            all_i = torch.empty((world * per_rank, max_el), dtype=dt, device=dev)
            dist.all_gather_into_tensor(all_i, my_i)
            ev_i1.record()
        self._events.append(("exchange_images", ev_i0, ev_i1))

        # ---- SIFT on the owned images (8-bit: the caller's tensors are read until exchange() queries the counts)
        def sift():
            if not mine:
                return None
            ws, hs = [shapes[k][1] for k in mine], [shapes[k][0] for k in mine]
            if rgb8:
                return eng.sift_detect_batch_rgb8_ptr([owned_pix[k].data_ptr() for k in mine], ws, hs,
                                                      [own_ch[k] for k in mine], params, device=True)
            return eng.sift_detect_batch_ptr([owned[k].data_ptr() for k in mine], ws, hs, params, device=True)
        fs_local = self._timed("sift", sift)

        # ---- C1: all-gather of the descriptor sets.  The counts' all-reduce also carries each image's channel
        # count (run_rgb8), which every rank's strip needs and only the owner knows.
        def exchange():
            arr = np.zeros(2 * n_images, np.int64)
            for q, k in enumerate(mine):
                arr[k] = fs_local.count(q)
                arr[n_images + k] = own_ch.get(k, 3)
            counts_t = torch.from_numpy(arr).to(dev)
            dist.all_reduce(counts_t)
            both = [int(c) for c in counts_t.tolist()]
            counts, chans = both[:n_images], both[n_images:]
            rows = [sum(counts[k] for k in owners[r]) for r in range(world)]
            pad = max(max(rows), 1)
            my_d = torch.empty((pad, 128), dtype=torch.float32, device=dev)
            my_c = torch.empty((pad, 2), dtype=torch.float64, device=dev)
            if mine:
                fs_local.export_all_dev(my_c.data_ptr(), my_d.data_ptr())      # one launch for all owned images
            all_d = torch.empty((world * pad, 128), dtype=torch.float32, device=dev)
            all_c = torch.empty((world * pad, 2), dtype=torch.float64, device=dev)
            dist.all_gather_into_tensor(all_d, my_d)
            dist.all_gather_into_tensor(all_c, my_c)
            pd, pc = [0] * n_images, [0] * n_images
            for r in range(world):
                off = 0
                for k in owners[r]:
                    pd[k] = all_d.data_ptr() + (r * pad + off) * 512
                    pc[k] = all_c.data_ptr() + (r * pad + off) * 16
                    off += counts[k]
            fs_all = eng.featureset_import_dev(counts, pd, pc)
            return fs_all, counts, chans, (all_d, all_c, my_d, my_c)
        fs_all, counts, chans, keep = self._timed("exchange_descriptors", exchange)
        if fs_local is not None:
            fs_local.free()

        # ---- dealt pair tasks
        dealt = deal_pairs(pairs, counts, world)
        tasks = dealt[rank]
        results = self._timed("match", lambda: eng.match_pairs(fs_all, [pairs[t] for t in tasks], params) if tasks else [])

        # ---- match lists to rank 0, part 1: the largest per-rank total (one scalar all-reduce, read back through
        # pinned memory behind an event so that waiting for it does not wait for the blend queued after it)
        ntask = max(max(len(d) for d in dealt), 1)
        tot = sum(len(m) for m in results) if tasks else 0
        t_max = torch.tensor([tot], dtype=torch.int32, device=dev)
        dist.all_reduce(t_max, op=dist.ReduceOp.MAX)
        t_host = self._pinned("scalar", 1)
        t_host[:1].copy_(t_max, non_blocking=True)
        ev_tot = torch.cuda.Event()
        ev_tot.record()

        # part 2 (after the blend and C2 are queued): ONE all-gather of [number of matches per dealt task ...,
        # (i, j) ...] padded to that total, through pinned staging both ways.  (Padding to the a-priori bound
        # min(N_i, N_j) per pair needs no scalar round trip but moves ~14x the bytes of the real lists on a
        # 38-image all-pairs job at 4 ranks.)
        def gather_lists():
            stage = self._pinned("send", ntask + 2 * max(tot, 1))
            host = stage.numpy()
            pack_match_lists(results if tasks else [], ntask, host)
            ev_tot.synchronize()
            pad = ntask + 2 * max(int(t_host[0]), 1)
            if stage.numel() < pad:                              # another rank has more: same content, longer buffer
                bigger = self._pinned("send2", pad)
                bigger[:ntask + 2 * tot].copy_(stage[:ntask + 2 * tot])
                stage, host = bigger, bigger.numpy()
            host[ntask + 2 * tot:pad] = 0
            my = torch.empty(pad, dtype=torch.int32, device=dev)
            my.copy_(stage[:pad], non_blocking=True)
            allm = torch.empty(world * pad, dtype=torch.int32, device=dev)
            dist.all_gather_into_tensor(allm, my)
            if rank != 0:
                torch.cuda.current_stream().synchronize()      # the staging buffer is reused by the next job
                return None
            back = self._pinned("recv", world * pad)
            back[:world * pad].copy_(allm, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            return unpack_match_lists(back.numpy(), dealt, ntask, pad, len(pairs))

        # ---- strip of the canvas, then C2
        main.wait_stream(side)                              # the image exchange has landed
        tw, th = max(it[2] for it in items), max(it[3] for it in items)
        rows_per = (th + world - 1) // world
        row0, row1 = min(th, rank * rows_per), min(th, (rank + 1) * rows_per)
        strip = torch.empty((rows_per, tw, 3), dtype=torch.float32, device=dev)
        bparams = self.blend_params

        def blend_strip():
            el = 1 if rgb8 else 4
            src_ptrs = [0] * n_images
            for r in range(world):
                for q, k in enumerate(owners[r]):
                    src_ptrs[k] = all_i.data_ptr() + (r * per_rank + q) * max_el * el
            if rgb8:
                eng.blend_rows_rgb8_dev(src_ptrs, chans, shapes, items, geom, strip.data_ptr(), tw, th, row0, row1,
                                        bands, bparams)
            else:
                eng.blend_rows_dev(src_ptrs, shapes, items, geom, strip.data_ptr(), tw, th, row0, row1, bands, bparams)
        self._timed("blend_strip", blend_strip)
        mosaic = torch.empty((world * rows_per, tw, 3), dtype=torch.float32, device=dev)
        self._timed("gather_strips", lambda: dist.all_gather_into_tensor(mosaic, strip))
        # the match lists last: their host work (staging, parsing) runs while the GPU blends and gathers the strips
        # — the composite depends on the images and the caller's geometry only
        matches = self._timed("gather_matches", gather_lists)
        torch.cuda.current_stream().synchronize()
        side.synchronize()
        self.ms = {}
        for name, e0, e1 in self._events:
            self.ms[name] = self.ms.get(name, 0.0) + e0.elapsed_time(e1)
        fs_all.free()
        del keep, my_i, all_i
        return matches, mosaic[:th]
