"""Host-side mirror of the reference's orchestration for the hot path.

`Stitcher.build()` follows Stitcher::build() (stitch/stitcher.cc:32-64):
calc_feature() (stitcherbase.cc:9-27) -> linear/pairwise match
(stitcher.cc:96-136) -> ConnectedImages::blend() (stitcher_image.cc:116-155).
The geometry in between (RANSAC, camera estimation, bundle adjustment) is host
code outside the hot path (SURVEY.md §8 scope): the caller supplies the
per-image inverse homographies and ranges it produced, exactly the numbers the
reference's blend lambda closes over.

Everything heavy is one C-ABI call into libpano_b200.so; this class only owns
the device buffers so that images are uploaded once per build and reused by the
feature and blend stages.
"""
from __future__ import annotations

import numpy as np

from ._abi import default_params
from .capi import (PIX_FORMATS, PIX_RGB, PIX_RGBA, PIX_RGB_PLANAR, SRC_F32_HOST, SRC_RGB8_DEV, SRC_RGB8_HOST, Engine,
                   pix_format)


from .synth import all_pairs, ordered_pairs  # noqa: F401  (task lists live with the workload generator)


class Stitcher:
    def __init__(self, engine: Engine, params=None, overlap_blend: bool = True):
        """overlap_blend: the composite depends on the images and the caller's geometry only, not
        on the features (the geometry in between is host code), so it runs on a second context /
        stream of the same device, ordered with events (see run_device); results are unchanged."""
        self.eng = engine
        self.params = params or default_params()
        self._aux = None
        self._overlap = overlap_blend
        self._ev_in = self._ev_blend = None
        self._d_imgs = None      # device block holding all input images
        self._d_out = None
        self._shapes = None
        self._offs = None
        self._out_shape = None

    # -- device buffers, (re)allocated only when the workload shape changes
    def _ensure(self, shapes, out_wh):
        if self._shapes != shapes:
            self.release_images()
            offs, total = [], 0
            for (h, w) in shapes:
                offs.append(total)
                total += (h * w * 3 * 4 + 255) // 256 * 256
            self._d_imgs = self.eng.dev_alloc(max(total, 256))
            self._shapes, self._offs = list(shapes), offs
        if self._out_shape != out_wh:
            if self._d_out:
                self.eng.dev_free(self._d_out)
            self._d_out = self.eng.dev_alloc(max(out_wh[0] * out_wh[1] * 3 * 4, 256))
            self._out_shape = out_wh

    def release_images(self):
        if self._d_imgs:
            self.eng.dev_free(self._d_imgs)
            self._d_imgs = None
            self._shapes = None

    def close(self):
        self.release_images()
        if self._d_out:
            self.eng.dev_free(self._d_out)
            self._d_out = None
            self._out_shape = None
        if self._aux is not None:
            self._aux.sync()
            Engine.event_destroy(self._ev_in)
            Engine.event_destroy(self._ev_blend)
            self._aux.close()
            self._aux = None

    def _aux_engine(self):
        if self._aux is None:
            self._aux = Engine(self.eng.device)
            self._ev_in = self.eng.event_create()
            self._ev_blend = self._aux.event_create()
        return self._aux

    def image_ptrs(self):
        return [self._d_imgs + o for o in self._offs]

    # -- stages on device-resident inputs (bench `value` leg)
    def upload(self, host_ptrs, shapes, out_wh):
        """host_ptrs: raw pointers of PINNED H×W×3 float32 buffers."""
        self._ensure(list(shapes), tuple(out_wh))
        for p, o, (h, w) in zip(host_ptrs, self._offs, shapes):
            self.eng.dev_upload_async(self._d_imgs + o, p, h * w * 3 * 4)

    def run_device(self, pairs, items, geom, bands=0, want_matches=False):
        """SIFT + match + blend on the images already in HBM.  Returns
        (featureset, matches-or-total)."""
        shapes = self._shapes
        ptrs = self.image_ptrs()
        fs = self.eng.sift_detect_batch_ptr(ptrs, [s[1] for s in shapes], [s[0] for s in shapes], self.params,
                                            device=True)
        if self._overlap:
            # The composite waits for SIFT's last kernel.  Queued ahead of SIFT, its grid filled every SM and
            # SIFT's kernels waited behind it; waiting for the images only, it slowed SIFT by more than it
            # saved.  Behind SIFT it runs while the host reads the feature counts and plans the matcher.
            aux = self._aux_engine()
            self.eng.event_record(self._ev_in)
            aux.event_wait(self._ev_in)
            aux.blend_dev(ptrs, shapes, items, geom, self._d_out, self._out_shape[0], self._out_shape[1], bands, self.params)
            aux.event_record(self._ev_blend)
        if want_matches:
            m = self.eng.match_pairs(fs, pairs, self.params)
        else:
            m = self.eng.match_pairs_dev(fs, pairs, self.params)
        if self._overlap:
            self.eng.event_wait(self._ev_blend)         # the mosaic is complete in main-stream order
        else:
            self.eng.blend_dev(ptrs, shapes, items, geom, self._d_out, self._out_shape[0], self._out_shape[1], bands,
                               self.params)
        return fs, m

    # -- the end-to-end call a user makes: host images in, host mosaic + matches out
    def build(self, host_ptrs, shapes, pairs, items, geom, out_host_ptr, bands=0):
        out_w = max(it[2] for it in items)
        out_h = max(it[3] for it in items)
        self.upload(host_ptrs, shapes, (out_w, out_h))
        fs, matches = self.run_device(pairs, items, geom, bands, want_matches=True)
        self.eng.dev_download_async(out_host_ptr, self._d_out, out_w * out_h * 3 * 4)
        self.eng.sync()
        fs.free()
        return matches

    def build_numpy(self, imgs, pairs, items, geom, bands=0):
        """Convenience for tests: numpy in/out (pageable memory; slower)."""
        imgs = [np.ascontiguousarray(im, np.float32) for im in imgs]
        out_w = max(it[2] for it in items)
        out_h = max(it[3] for it in items)
        out = np.empty((out_h, out_w, 3), np.float32)
        m = self.build([im.ctypes.data for im in imgs], [im.shape[:2] for im in imgs], pairs, items, geom,
                       out.ctypes.data, bands)
        return m, out


class PipelinedStitcher:
    """Throughput form of Stitcher.build(): consecutive stitch jobs overlap on the
    device.  Three contexts share the GPU — upload, compute and download, each with
    its own stream — ordered by events, so job i+1's images cross PCIe while job i
    runs SIFT/match/blend and job i-1's mosaic streams back (PCIe is full duplex).

        slot = ps.stage(host_ptrs, shapes, out_wh)     # enqueue the H2D copies
        job  = ps.run(slot, pairs, items, geom, out_host_ptr)   # compute + enqueue D2H
        matches = ps.wait(job)                          # host mosaic + matches ready

    Call stage() for the NEXT job before run() of the current one: run() blocks the
    host while the match lists come back, and that is when the next upload flies.
    """

    def __init__(self, device: int, params=None, depth: int = 2, rgb8: bool = False, crop: bool = True,
                 in_format: str = "rgb", out_format: str = "rgb"):
        """rgb8: the host side speaks the reference's FILE formats instead of Mat32f —
        decoded 8-bit pixels in (what read_img starts from, imgio.cc:72) and the 8-bit
        mosaic out (what write_rgb saves, imgio.cc:98-113, after crop() when `crop`,
        main.cc:226-229) — so 3 B/px cross PCIe each way instead of 12.  SIFT and the blend
        read the 8-bit pixels directly (each tap converted as read_img converts it), so no
        f32 copy of an image exists on the device; the output conversion runs there with
        the reference's arithmetic.  The output buffer then
        holds a 256-byte header (int32 x0, y0, width, height of the crop rectangle)
        followed by height*width*3 packed bytes.

        in_format / out_format (rgb8 only) select the layouts of the reference's codecs
        instead of interleaved RGB: "rgba" is lodepng's (read_png's input, imgio.cc:43-61;
        write_png's output with alpha 255, h*w*4 bytes), "planar" is CImg<unsigned char>'s
        (three h×w planes R, G, B: read_img's other path and write_rgb's image).  The mosaic
        is the interleaved path's, re-laid out (unpack_rgb8_mosaic reads it back)."""
        if in_format not in ("rgb", "rgba", "planar") or out_format not in ("rgb", "rgba", "planar"):
            raise ValueError(f"in_format / out_format: 'rgb', 'rgba' or 'planar', not {in_format!r} / {out_format!r}")
        if not rgb8 and (in_format, out_format) != ("rgb", "rgb"):
            raise ValueError("in_format / out_format need rgb8=True")
        self.params = params or default_params()
        self.up = Engine(device)
        self.cmp = Engine(device)
        self.dn = Engine(device)
        self.depth = depth
        self.rgb8 = rgb8
        self.crop = crop
        self.in_code, self.out_code = PIX_FORMATS[in_format], PIX_FORMATS[out_format]
        self.in_bpp = 4 if self.in_code == PIX_RGBA else 3
        self.out_bpp = 4 if self.out_code == PIX_RGBA else 3
        self.slots = [dict(imgs=None, out=None, shapes=None, offs=None, out_wh=None, pix=None, pix_offs=None, out8=None,
                           ev_up=self.up.event_create(), ev_cmp=self.cmp.event_create(),
                           ev_dn=self.dn.event_create(), busy=False) for _ in range(depth)]
        self._next = 0

    def _ensure(self, s, shapes, out_wh):
        realloc = False
        if s["shapes"] != shapes:
            realloc = True
            # one device block per slot: the f32 images, or with rgb8 the 8-bit pixels that SIFT and the
            # blend read directly
            key, offs_key, px = ("pix", "pix_offs", self.in_bpp) if self.rgb8 else ("imgs", "offs", 12)
            if s[key]:
                self.cmp.dev_free(s[key])
            offs, total = [], 0
            for (h, w) in shapes:
                offs.append(total)
                total += (h * w * px + 255) // 256 * 256
            s[key] = self.cmp.dev_alloc(max(total, 256))
            s["shapes"], s[offs_key] = list(shapes), offs
        if s["out_wh"] != out_wh:
            if s["out"]:
                self.cmp.dev_free(s["out"])
            s["out"] = self.cmp.dev_alloc(max(out_wh[0] * out_wh[1] * 3 * 4, 256))
            if self.rgb8:
                if s["out8"]:
                    self.cmp.dev_free(s["out8"])
                s["out8"] = self.cmp.dev_alloc(self.out_bytes(out_wh))
            s["out_wh"] = tuple(out_wh)
            realloc = True
        if realloc:
            # The buffers come stream-ordered from the compute context's pool, but the upload
            # stream writes them first: a block the pool hands out may still be in use by work
            # queued on cmp (the other slot's featureset, a SIFT arena freed in stream order).
            # Drain cmp so that the allocation is complete and the block idle before `up` touches it.
            self.cmp.sync()

    RGB8_HEADER = 256

    def out_bytes(self, out_wh) -> int:
        """Size of the host buffer run() fills for a canvas of out_wh."""
        if self.rgb8:
            return self.RGB8_HEADER + out_wh[0] * out_wh[1] * self.out_bpp
        return out_wh[0] * out_wh[1] * 3 * 4

    def in_bytes(self, shapes) -> int:
        return sum(h * w * (self.in_bpp if self.rgb8 else 12) for (h, w) in shapes)

    def stage(self, host_ptrs, shapes, out_wh) -> int:
        k = self._next
        self._next = (self._next + 1) % self.depth
        s = self.slots[k]
        if s["busy"]:
            Engine.event_sync(s["ev_dn"])          # the slot's previous job has fully left the device
            s["busy"] = False
        self._ensure(s, list(shapes), tuple(out_wh))
        self.up.event_wait(s["ev_cmp"])            # its previous compute no longer reads these images
        if self.rgb8:
            for p, o, (h, w) in zip(host_ptrs, s["pix_offs"], shapes):
                self.up.dev_upload_async(s["pix"] + o, p, h * w * self.in_bpp)
        else:
            for p, o, (h, w) in zip(host_ptrs, s["offs"], shapes):
                self.up.dev_upload_async(s["imgs"] + o, p, h * w * 3 * 4)
        self.up.event_record(s["ev_up"])
        return k

    def run(self, k: int, pairs, items, geom, out_host_ptr, bands: int = 0):
        s = self.slots[k]
        shapes = s["shapes"]
        ws, hs = [q[1] for q in shapes], [q[0] for q in shapes]
        self.cmp.event_wait(s["ev_up"])
        if self.rgb8:
            ptrs, chans = [s["pix"] + o for o in s["pix_offs"]], [self.in_code] * len(shapes)
            fs = self.cmp.sift_detect_batch_rgb8_ptr(ptrs, ws, hs, chans, self.params, device=True)
        else:
            ptrs = [s["imgs"] + o for o in s["offs"]]
            fs = self.cmp.sift_detect_batch_ptr(ptrs, ws, hs, self.params, device=True)
        matches = self.cmp.match_pairs(fs, pairs, self.params)       # host waits here; copies keep flowing
        self.cmp.event_wait(s["ev_dn"])                               # previous mosaic of this slot is out
        ow, oh = s["out_wh"]
        if self.rgb8:
            self.cmp.blend_rgb8_dev(ptrs, chans, shapes, items, geom, s["out"], ow, oh, bands, self.params)
        else:
            self.cmp.blend_dev(ptrs, shapes, items, geom, s["out"], ow, oh, bands, self.params)
        if self.rgb8:
            if self.crop:
                self.cmp.crop_rect_dev(s["out"], ow, oh, s["out8"])
            rect = s["out8"] if self.crop else 0
            if self.out_code == PIX_RGB:
                self.cmp.mat32f_to_rgb8_dev(s["out"], ow, oh, rect, s["out8"] + self.RGB8_HEADER)
            else:
                self.cmp.mat32f_to_pix8_dev(s["out"], ow, oh, rect, self.out_code, s["out8"] + self.RGB8_HEADER)
        self.cmp.event_record(s["ev_cmp"])
        fs.free()
        self.dn.event_wait(s["ev_cmp"])
        if self.rgb8:
            self.dn.dev_download_async(out_host_ptr, s["out8"], self.out_bytes((ow, oh)))
        else:
            self.dn.dev_download_async(out_host_ptr, s["out"], ow * oh * 3 * 4)
        self.dn.event_record(s["ev_dn"])
        s["busy"] = True
        return (k, matches)

    def wait(self, job):
        k, matches = job
        Engine.event_sync(self.slots[k]["ev_dn"])
        self.slots[k]["busy"] = False
        return matches

    def close(self):
        for e in (self.up, self.cmp, self.dn):
            try:
                e.sync()
            except Exception:
                pass
        for s in self.slots:
            if s["imgs"]:
                self.cmp.dev_free(s["imgs"])
            if s["out"]:
                self.cmp.dev_free(s["out"])
            for key in ("pix", "out8"):
                if s[key]:
                    self.cmp.dev_free(s[key])
            for key in ("ev_up", "ev_cmp", "ev_dn"):
                Engine.event_destroy(s[key])
        self.slots = []
        for e in (self.up, self.cmp, self.dn):
            e.close()


def unpack_rgb8_mosaic(buf: np.ndarray, out_wh, cropped: bool = True, out_format: str = "rgb"):
    """View of the 8-bit mosaic PipelinedStitcher(rgb8=True).run() wrote into `buf`
    (uint8, out_bytes long).  Returns (rect (x0, y0, w, h), uint8 view): H×W×3, or H×W×4 for
    out_format "rgba", or 3×H×W for "planar"."""
    hdr = PipelinedStitcher.RGB8_HEADER
    if cropped:
        x0, y0, w, h = (int(v) for v in buf[:16].view(np.int32))
    else:
        x0, y0, w, h = 0, 0, out_wh[0], out_wh[1]
    code = PIX_FORMATS[out_format]
    if code == PIX_RGB_PLANAR:
        return (x0, y0, w, h), buf[hdr:hdr + w * h * 3].reshape(3, h, w)
    bpp = 4 if code == PIX_RGBA else 3
    return (x0, y0, w, h), buf[hdr:hdr + w * h * bpp].reshape(h, w, bpp)


def mosaic_rgb8_strips(engine: Engine, items, geom, bands, sources, strip_rows, window=1, out_format="rgb",
                       crop=True, params=None, kind=None, channels=3, shapes=None, fmt=None):
    """ConnectedImages::blend() + crop() + write_rgb's conversion strip by strip, without the f32 mosaic.

    Each strip of `strip_rows` canvas rows is a row-strip blend stream fed only the sources it needs, `window` of
    them per add (None: all in one add).  Its f32 rows go through the crop scan and into an uncropped 8-bit canvas,
    which is cropped at the end.  sources: numpy arrays (host uint8 read in layout `fmt`, or float32 H×W×3), or
    pointers of source kind `kind` with PANO_PIX_* code `channels` and `shapes` [(h, w)].  Device memory holds
    one strip's blend state and f32 rows, two windows of sources, and 3 + 3 (4 for "rgba") bytes per canvas pixel.
    Returns (rect or None, pixels) as Engine.crop_write_pix8 does: the same bytes as crop_write_pix8 on the
    mosaic of Engine.blend."""
    n = len(items)
    if shapes is None:
        shapes = [pix_format(a, fmt)[1:] if a.dtype == np.uint8 and fmt is not None else a.shape[:2] for a in sources]
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    code = PIX_FORMATS[out_format]
    bpp = 4 if code == PIX_RGBA else 3
    window = window or n
    d_strip = engine.dev_alloc(min(strip_rows, oh) * ow * 12)
    d_rgb = engine.dev_alloc(ow * oh * 3)
    d_out = engine.dev_alloc(ow * oh * bpp)
    d_rect = engine.dev_alloc(256)
    scan = engine.crop_scan(ow, oh) if crop else None
    try:
        for r0 in range(0, oh, strip_rows):
            r1 = min(oh, r0 + strip_rows)
            s = engine.blend_stream_rows(shapes, items, geom, r0, r1, bands, params)
            try:
                need = s.needs()
                batch, used = [], 0
                for k in range(n):          # adds of `window` needed images each, unneeded ones passed as None
                    batch.append(sources[k] if need[k] else None)
                    used += int(need[k])
                    if used == window or k == n - 1:
                        s.add(batch, kind, channels, fmt)
                        batch, used = [], 0
                s.finish_dev(d_strip)
            finally:
                s.close()
            if scan is not None:
                scan.add_dev(d_strip, r1 - r0)
            engine.mat32f_to_rgb8_dev(d_strip, ow, r1 - r0, 0, d_rgb + r0 * ow * 3)
        rect = None
        if scan is not None:
            rect = scan.rect()
            engine.dev_upload(d_rect, rect)
        engine.rgb8_crop_to_pix8_dev(d_rgb, ow, oh, d_rect if crop else 0, code, d_out)
        cw, ch = (int(rect[2]), int(rect[3])) if crop else (ow, oh)
        px = np.empty(cw * ch * bpp, np.uint8)
        if px.size:
            engine.dev_download(px, d_out)
    finally:
        if scan is not None:
            scan.close()
        for d in (d_strip, d_rgb, d_out, d_rect):
            engine.dev_free(d)
    return rect, (px.reshape(3, ch, cw) if code == PIX_RGB_PLANAR else px.reshape(ch, cw, bpp))


_PIX_BYTES = {1: 1, 3: 3, PIX_RGBA: 4, PIX_RGB_PLANAR: 3}


def _sweep_sources(sources, n, kind, formats, shapes, fmt):
    """A sweep's sources as (kind, formats, shapes, sources, bytes): numpy arrays (host, pageable: uint8 read in
    layout `fmt`, one value or one per image, or float32 H×W×3), or pointers of kind `kind` with PANO_PIX_* codes
    `formats` (None: 3) and `shapes` [(h, w)].  The sources returned are the C-contiguous arrays the sweep reads
    (copies of the others) or the pointers: the caller holds them until the sweep has run."""
    if kind is None:
        arrs = [np.ascontiguousarray(a) for a in sources]
        u8 = arrs[0].dtype == np.uint8
        if u8:
            info = [pix_format(a, f) for a, f in zip(arrs, fmt if isinstance(fmt, (list, tuple)) else [fmt] * n)]
            formats, shapes = [c for c, _, _ in info], [(h, w) for _, h, w in info]
        else:
            formats, shapes = [3] * n, [a.shape[:2] for a in arrs]
        kind = SRC_RGB8_HOST if u8 else SRC_F32_HOST
        return kind, formats, shapes, arrs, [a.nbytes for a in arrs]
    u8 = kind in (SRC_RGB8_DEV, SRC_RGB8_HOST)
    formats = list(formats) if formats is not None else [3] * n
    nbytes = [h * w * (_PIX_BYTES[f] if u8 else 12) for (h, w), f in zip(shapes, formats)]
    return kind, formats, shapes, list(sources), nbytes


def _run_sweep(engine, sweep, srcs, formats, kind, ow, oh, out_format, crop, stats):
    """Runs every strip of `sweep` on srcs (_sweep_sources' sources, alive for the whole call), then its finish_dev;
    returns (rect or None, pixels) and frees the sweep."""
    ptrs = [q.ctypes.data if isinstance(q, np.ndarray) else q for q in srcs]
    code = PIX_FORMATS[out_format]
    bpp = 4 if code == PIX_RGBA else 3
    d_out = engine.dev_alloc(max(ow * oh * bpp, 256))
    try:
        while True:
            st, want = sweep.next()
            if st < 0:
                break
            sweep.strip([q if w else 0 for q, w in zip(ptrs, want)], formats, kind)
        rect = sweep.finish_dev(code, d_out)
        cw, ch = int(rect[2]), int(rect[3])
        px = np.empty(cw * ch * bpp, np.uint8)
        if px.size:
            engine.dev_download(px, d_out)
        if stats is not None:
            stats["uploads"], stats["upload_bytes"], stats["retained_high"] = sweep.stats()
    finally:
        sweep.close()
        engine.dev_free(d_out)
    return (rect if crop else None), (px.reshape(3, ch, cw) if code == PIX_RGB_PLANAR else px.reshape(ch, cw, bpp))


def mosaic_rgb8_sweep(engine: Engine, items, geom, bands, sources, strip_rows, keep_bytes, out_format="rgb", crop=True,
                      params=None, kind=None, formats=None, shapes=None, fmt=None, stats=None):
    """mosaic_rgb8_strips' bytes from one blend sweep (Engine.blend_sweep): the strips run top to bottom and each
    source is handed over once while a later strip still reads it, keeping at most keep_bytes of sources between
    strips (capi.SIZE_MAX: no limit; 0 hands over every source each strip reads).

    sources: numpy arrays (host, pageable: uint8 read in layout `fmt`, one value or one per image, or float32
    H×W×3), or pointers of source kind `kind` with PANO_PIX_* codes `formats` (one per image; None: 3) and `shapes`
    [(h, w)].  Device memory holds one strip's blend state and f32 rows, two sources in the upload ring, the kept
    sources, and 3 + 3 (4 for "rgba") bytes per canvas pixel.  stats: a dict that receives
    "uploads", "upload_bytes" and "retained_high" (pano_blend_sweep_stats).  Returns (rect or None, pixels) as
    mosaic_rgb8_strips does."""
    n = len(items)
    kind, formats, shapes, srcs, nbytes = _sweep_sources(sources, n, kind, formats, shapes, fmt)
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    sweep = engine.blend_sweep(shapes, items, geom, strip_rows, keep_bytes, bands, params, crop, nbytes)
    return _run_sweep(engine, sweep, srcs, formats, kind, ow, oh, out_format, crop, stats)


def cylinder_mosaic_rgb8_sweep(engine: Engine, items, geom, h_factor, corr_inv, bands, sources, strip_rows, keep_bytes,
                               out_format="rgb", crop=True, params=None, kind=None, formats=None, shapes=None, fmt=None,
                               stats=None):
    """Cylinder mode's output, write_rgb(crop(CylinderStitcher::build())), from one cylinder sweep
    (Engine.blend_sweep_cyl): each strip of the corrected canvas blends the band of mosaic rows its perspective
    correction reads, straight from the UNWARPED sources, and corrects its rows from it; no f32 mosaic of the whole
    canvas is made.  items / geom: the warped images' (as for Engine.blend_stream_cyl); corr_inv:
    perspective_correction's inv (3×3).  sources, kind, formats, shapes (the unwarped sources'), fmt, keep_bytes,
    out_format, crop and stats as for mosaic_rgb8_sweep.  Device memory holds the tallest band's blend state and
    f32 rows, one strip's f32 rows, two sources in the upload ring, the kept sources, the warps' column tables and
    3 + 3 (4 for "rgba") bytes per canvas pixel.  Returns (rect or None, pixels) as mosaic_rgb8_sweep does."""
    n = len(items)
    kind, formats, shapes, srcs, nbytes = _sweep_sources(sources, n, kind, formats, shapes, fmt)
    ow, oh = max(it[2] for it in items), max(it[3] for it in items)
    sweep = engine.blend_sweep_cyl(shapes, items, geom, h_factor, corr_inv, strip_rows, keep_bytes, bands, params,
                                   crop, nbytes)
    return _run_sweep(engine, sweep, srcs, formats, kind, ow, oh, out_format, crop, stats)


class StitchLanes:
    """Several PipelinedStitcher lanes on ONE GPU, one host thread per lane.

    A single lane leaves the compute stream idle whenever its host thread is between
    two dependent phases of a job (feature counts -> match plan -> match lists ->
    blend launch) and whenever a tiny metadata move waits on a busy PCIe link.  With
    two lanes the other job's kernels fill those gaps (ctypes releases the GIL inside
    every engine call, so the lanes' host threads run concurrently).

        lanes = StitchLanes(device, params, lanes=2, rgb8=True)
        results = lanes.map(jobs)     # jobs[i] = (host_ptrs, shapes, out_wh, pairs, items, geom, out_host_ptr, bands)
    """

    def __init__(self, device: int, params=None, lanes: int = 2, depth: int = 2, rgb8: bool = False, crop: bool = True,
                 in_format: str = "rgb", out_format: str = "rgb"):
        self.lanes = [PipelinedStitcher(device, params, depth=depth, rgb8=rgb8, crop=crop, in_format=in_format,
                                        out_format=out_format) for _ in range(lanes)]
        self.done_times = []       # perf_counter() at which each job of the last map() came back (diagnostics)

    def out_bytes(self, out_wh):
        return self.lanes[0].out_bytes(out_wh)

    def in_bytes(self, shapes):
        return self.lanes[0].in_bytes(shapes)

    @staticmethod
    def _run_lane(ps, jobs, results, errors, done=None):
        import time
        try:
            if not jobs:
                return
            it = iter(jobs)
            idx, job = next(it)
            slot = ps.stage(job[0], job[1], job[2])
            pending = None
            while job is not None:
                nxt = next(it, None)
                nslot = ps.stage(nxt[1][0], nxt[1][1], nxt[1][2]) if nxt is not None else None
                handle = ps.run(slot, job[3], job[4], job[5], job[6], job[7])
                if pending is not None:
                    results[pending[0]] = ps.wait(pending[1])
                    if done is not None:
                        done[pending[0]] = time.perf_counter()
                pending = (idx, handle)
                if nxt is None:
                    break
                (idx, job), slot = nxt, nslot
            results[pending[0]] = ps.wait(pending[1])
            if done is not None:
                done[pending[0]] = time.perf_counter()
        except Exception as ex:  # surfaced by map()
            errors.append(ex)

    def map(self, jobs):
        """Runs the jobs (in order within a lane, job i on lane i mod L); returns their match lists."""
        import threading
        jobs = list(jobs)
        results = [None] * len(jobs)
        errors = []
        done = [0.0] * len(jobs)
        L = len(self.lanes)
        threads = [threading.Thread(target=self._run_lane, args=(self.lanes[q], [(i, j) for i, j in enumerate(jobs) if i % L == q],
                                                                 results, errors, done)) for q in range(L)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        self.done_times = done
        return results

    def close(self):
        for ps in self.lanes:
            ps.close()
        self.lanes = []
