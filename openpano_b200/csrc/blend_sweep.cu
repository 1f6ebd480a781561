// blend_sweep.cu — the row strips of the canvas, top to bottom, with every source handed over once while it stays
// in use (pano_blend_sweep_*, pano_b200.h).
//
// A row-strip stream (pano_blend_stream_create_rows) holds two windows of sources at most, so a strip-by-strip
// writer uploads a source once for every strip it reaches.  The strips run in order and the images each one reads
// are known up front (blend_strip_reads), so the sweep plans the whole access sequence at creation: a source read
// again later is kept on the device, within keep_bytes, evicting the kept source whose next use is farthest away.
// Each strip then runs an ordinary row-strip stream over device pointers (its kernels, its bits), feeds the crop
// scan and converts its rows into the 8-bit canvas, as stitcher.mosaic_rgb8_strips does.
//
// A cylinder sweep (pano_blend_sweep_create_cyl) runs the strips of cylinder mode's perspective-corrected canvas:
// each strip blends the band of mosaic rows its correction reads (persp_band) as a cylinder row stream from the
// unwarped sources, then corrects its own rows from that band (persp_correct_rows); the plan is made over the
// bands' read sets, and everything after the correction is the plain sweep's.
//
// Host sources go one per window through an UploadRing on the ring's copy stream, so each crosses PCIe while the
// kernels of the window before it run, this strip's or the previous one's.  A kept one is then copied on the ctx
// stream into a block of its own, freed in stream order when the plan drops it: every reader and the free are on the
// ctx stream, so the ring's ordering is the only cross-stream ordering there is.
#include "common.cuh"
#include "blend_rows.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

namespace {

struct SweepPlan {
  int n = 0, strips = 0;
  std::vector<unsigned char> reads, uploads, kept, held;   // strips × n; held: kept once the strip has run
  std::vector<int> band;           // strips × 2: the canvas rows [b0, b1) each strip blends
  long long n_uploads = 0;
  unsigned long long upload_bytes = 0, retained_high = 0;
};

// Cylinder mode's perspective correction maps output pixel (j, i) to inv.trans2d(j, i) of the mosaic
// (cylstitcher.cc:171-179) and reads rows floor(y) and floor(y) + 1 there.  The map is projective: where z keeps
// one sign over the strip's pixels [0, w - 1] × [r0, r1 - 1], y is a linear-fractional function of the pixel
// and takes its extremes at the four corners, so the rows read lie in [floor(min y), floor(max y) + 1]; one row
// more on each side covers the float rounding of y and the last bits of the interior pixels' arithmetic.  Where
// z changes sign, is 0 or is not a number at a corner, the band is the whole mosaic.  Clamped to [0, h); b0 ==
// b1 when no row can be read.  The one statement of the rule: the plan (and so the runner) takes its bands here.
static void persp_band(const double inv[9], int w, int h, int r0, int r1, int* b0, int* b1) {
  double lo = INFINITY, hi = -INFINITY;
  int pos = 0, neg = 0;
  for (int c = 0; c < 4; ++c) {
    const double x = (c & 1) ? w - 1 : 0, y = (c & 2) ? r1 - 1 : r0;
    const double ry = inv[3] * x + inv[4] * y + inv[5] * 1.0;   // homography.hh:53-64, the kernel's order
    const double rz = inv[6] * x + inv[7] * y + inv[8] * 1.0;
    if (rz > 0) ++pos;
    else if (rz < 0) ++neg;
    const double denom = 1.0 / rz;
    const double yy = ry * denom;
    if (yy != yy) { pos = neg = 1; break; }
    lo = std::min(lo, yy); hi = std::max(hi, yy);
  }
  if (pos != 4 && neg != 4) { *b0 = 0; *b1 = h; return; }
  const double f0 = std::floor(lo) - 1, f1 = std::floor(hi) + 3;
  *b0 = f0 <= 0 ? 0 : f0 >= h ? h : (int)f0;
  *b1 = f1 <= 0 ? 0 : f1 >= h ? h : (int)f1;
  if (*b1 < *b0) *b1 = *b0;
}

// corr: the correction's inv for a cylinder sweep (strip s blends its band), else null (strip s blends its rows)
int make_plan(int n, const pano_blend_image* imgs, int bands, const pano_params* p, int ow, int oh, int strip_rows,
              const size_t* bytes, size_t keep, const double* corr, SweepPlan* pl) {
  if (n <= 0 || n > PANO_MAX_IMAGES || !imgs || !p || !bytes || bands < 0 || strip_rows < 1 || ow <= 0 || oh <= 0)
    return PANO_ERR_INVALID;
  int tw = 0, th = 0;
  for (int k = 0; k < n; ++k) {
    const pano_blend_image& s = imgs[k];
    if (s.w < 2 || s.h < 2 || s.x1 < s.x0 || s.y1 < s.y0 || s.x0 < 0 || s.y0 < 0 || bytes[k] == 0) return PANO_ERR_INVALID;
    tw = std::max(tw, s.x1); th = std::max(th, s.y1);
  }
  if (tw != ow || th != oh) return PANO_ERR_INVALID;
  const int halo = blend_halo(bands, p);
  if (halo < 0) return PANO_ERR_INVALID;
  const int S = (int)(((long long)oh + strip_rows - 1) / strip_rows);
  const size_t cells = (size_t)S * n;
  pl->n = n; pl->strips = S;
  pl->reads.assign(cells, 0); pl->uploads.assign(cells, 0); pl->kept.assign(cells, 0); pl->held.assign(cells, 0);
  pl->band.assign((size_t)S * 2, 0);
  for (int s = 0; s < S; ++s) {
    const int r0 = s * strip_rows, r1 = (int)std::min<long long>(oh, (long long)r0 + strip_rows);
    int b0 = r0, b1 = r1;
    if (corr) persp_band(corr, ow, oh, r0, r1, &b0, &b1);
    pl->band[2 * s] = b0; pl->band[2 * s + 1] = b1;
    if (b0 < b1)
      for (int k = 0; k < n; ++k) pl->reads[(size_t)s * n + k] = blend_strip_reads(imgs[k], bands, halo, oh, b0, b1);
  }
  // next_use[s * n + k]: the first strip after s that reads k, S for none
  std::vector<int> next_use(cells), nxt(n, S);
  for (int s = S - 1; s >= 0; --s)
    for (int k = 0; k < n; ++k) {
      next_use[(size_t)s * n + k] = nxt[k];
      if (pl->reads[(size_t)s * n + k]) nxt[k] = s;
    }
  std::vector<unsigned char> resident(n, 0);
  std::vector<int> cand;
  for (int s = 0; s < S; ++s) {
    const unsigned char* rd = &pl->reads[(size_t)s * n];
    const int* nu = &next_use[(size_t)s * n];
    for (int k = 0; k < n; ++k)
      if (rd[k] && !resident[k]) {
        pl->uploads[(size_t)s * n + k] = 1;
        ++pl->n_uploads;
        pl->upload_bytes += bytes[k];
      }
    // what may stay once the strip has run: resident or just read, and read again later
    cand.clear();
    unsigned long long total = 0;
    for (int k = 0; k < n; ++k)
      if ((resident[k] || rd[k]) && nu[k] < S) { cand.push_back(k); total += bytes[k]; }
    // evict the farthest next use first (ties: the higher index) until the rest fits
    std::sort(cand.begin(), cand.end(), [&](int a, int b) { return nu[a] != nu[b] ? nu[a] > nu[b] : a > b; });
    size_t q = 0;
    while (q < cand.size() && total > keep) total -= bytes[cand[q++]];
    std::fill(resident.begin(), resident.end(), 0);
    for (; q < cand.size(); ++q) resident[cand[q]] = 1;
    for (int k = 0; k < n; ++k) {
      pl->held[(size_t)s * n + k] = resident[k];
      pl->kept[(size_t)s * n + k] = pl->uploads[(size_t)s * n + k] && resident[k];
    }
    pl->retained_high = std::max(pl->retained_high, total);
  }
  return PANO_OK;
}

// One image's source while the plan keeps it: a block of the sweep's own (host sources) or the caller's device
// pointer.
struct Held {
  const void* ptr = nullptr;
  DevBuf<unsigned char> own;
  bool u8 = true;
  int fmt = PANO_PIX_RGB;
};

struct StreamFree { void operator()(pano_blend_stream* s) const { pano_blend_stream_free(s); } };
struct ScanFree { void operator()(pano_crop_scan* c) const { pano_crop_scan_free(c); } };

}  // namespace

struct pano_blend_sweep {
  Sticky st;
  int n = 0, bands = 0, ow = 0, oh = 0, rows = 0;
  pano_params p;
  pano_blend_geom g;
  std::vector<pano_blend_image> imgs;
  std::vector<int> src_w, src_h;   // each source's shape: imgs' for a plain sweep, the unwarped one for cylinder mode
  std::vector<size_t> bytes;
  SweepPlan plan;
  DevBuf<double> d_tab;            // projection tables of every strip (empty for flat)
  DevBuf<float> d_strip;           // one strip's f32 rows
  // cylinder sweeps (pano_blend_sweep_create_cyl), else empty: each strip blends its band of the mosaic from the
  // unwarped sources into d_band and corrects the strip's rows from it
  bool cyl = false;
  double corr[9];
  CylTabs ct;
  DevBuf<double> d_cyl_tab;        // ct.tabs, shared by every strip's stream
  DevBuf<float> d_band;            // the tallest band's f32 rows
  DevBuf<unsigned char> d_rgb;     // the 8-bit canvas
  DevBuf<int> d_rect;
  std::unique_ptr<pano_crop_scan, ScanFree> scan;
  std::vector<Held> held;
  int done = 0;
  long long uploads = 0;
  unsigned long long upload_bytes = 0, retained_high = 0;
  UploadRing ring;                 // last: its copy stream drains before the blocks above go
};

// The uploads of the previous strip are over: its pinned buffers are the caller's again.
static int sweep_wait_previous(pano_blend_sweep* s) {
  if (s->ring.copy)
    for (int b = 0; b < 2; ++b)
      if (int rc = s->st.cuda(cudaEventSynchronize(s->ring.ev_copied[b].get()),
                              "cudaEventSynchronize(s->ring.ev_copied[b].get())"))
        return rc;
  return PANO_OK;
}

// Blends rows [row0, row1) of the canvas for strip st as a row-strip stream into d_rows.  Windows are runs of
// sources of one kind and format, and a host source handed over starts a window of its own: it is uploaded through
// the ring just before that window is added, so the ring holds two sources and the next upload overlaps this
// window's kernels.  A kept one is then copied into a block of its own.  srcs / u8 / host / fmt / sz: the strip
// call's, checked.
static int sweep_blend_rows(pano_blend_sweep* s, int st, int row0, int row1, const void* const* srcs, bool u8,
                            bool host, const std::vector<int>& fmt, const std::vector<size_t>& sz, float* d_rows) {
  pano_ctx* ctx = s->st.ctx;
  const int n = s->n;
  const unsigned char* up = &s->plan.uploads[(size_t)st * n];
  const unsigned char* rd = &s->plan.reads[(size_t)st * n];
  const unsigned char* keep = &s->plan.kept[(size_t)st * n];
  std::vector<const void*> src(n, nullptr);   // null: not read, or a host source not uploaded yet
  std::vector<char> su8(n, 0);
  std::vector<int> sf(n, 3);
  for (int k = 0; k < n; ++k) {
    if (!rd[k]) continue;
    if (up[k]) {
      su8[k] = u8; sf[k] = fmt[k];
      if (host) continue;
      src[k] = srcs[k];
      if (keep[k]) { s->held[k] = Held(); s->held[k].ptr = srcs[k]; s->held[k].u8 = u8; s->held[k].fmt = fmt[k]; }
    } else {
      src[k] = s->held[k].ptr; su8[k] = s->held[k].u8; sf[k] = s->held[k].fmt;
    }
  }
  pano_blend_stream* raw = nullptr;
  int rc = s->cyl ? blend_stream_open_cyl(ctx, n, s->imgs.data(), &s->g, s->bands, &s->p, s->ow, s->oh, row0, row1,
                                          s->d_tab.get(), s->ct, s->d_cyl_tab.get(), &raw)
                  : blend_stream_open(ctx, n, s->imgs.data(), &s->g, s->bands, &s->p, s->ow, s->oh, row0, row1,
                                      s->d_tab.get(), &raw);
  if (rc) return rc;
  std::unique_ptr<pano_blend_stream, StreamFree> bs(raw);
  for (int k0 = 0; k0 < n;) {
    int k1 = k0, first = -1, upload = -1;
    for (; k1 < n; ++k1) {
      if (!rd[k1]) continue;
      const bool fresh = host && up[k1];
      if (first >= 0 && (fresh || su8[k1] != su8[first] || sf[k1] != sf[first])) break;
      if (first < 0) { first = k1; if (fresh) upload = k1; }
    }
    int slot = -1;
    if (upload >= 0) {
      if ((rc = s->ring.upload(ctx, "blend sweep", 1, &srcs[upload], &sz[upload], &src[upload], &slot))) return rc;
      if (keep[upload]) {
        Held& h = s->held[upload];
        h = Held();
        h.u8 = u8; h.fmt = fmt[upload];
        if ((rc = h.own.alloc(ctx, sz[upload]))) return rc;
        PANO_CUDA(ctx, cudaMemcpyAsync(h.own, src[upload], sz[upload], cudaMemcpyDeviceToDevice, ctx->stream));
        h.ptr = h.own.get();
      }
    }
    const bool w8 = first >= 0 && su8[first];
    if ((rc = pano_blend_stream_add(bs.get(), k0, k1 - k0, src.data() + k0, w8 ? PANO_SRC_RGB8_DEV : PANO_SRC_F32_DEV,
                                    first >= 0 ? sf[first] : 3)))
      return rc;
    if (slot >= 0) PANO_CUDA(ctx, s->ring.release(ctx, slot));
    k0 = k1;
  }
  return pano_blend_stream_finish_dev(bs.get(), d_rows);
}

// Runs strip st: its rows of the canvas into d_strip.  A plain sweep blends them; a cylinder sweep blends the
// strip's band of the mosaic into d_band (nothing when the band is empty) and corrects the strip's rows from it.
static int sweep_blend(pano_blend_sweep* s, int st, const void* const* srcs, bool u8, bool host,
                       const std::vector<int>& fmt, const std::vector<size_t>& sz) {
  const int row0 = s->plan.band[2 * st], row1 = s->plan.band[2 * st + 1];
  float* d_rows = s->cyl ? s->d_band.get() : s->d_strip.get();
  if (row0 < row1)
    if (int rc = sweep_blend_rows(s, st, row0, row1, srcs, u8, host, fmt, sz, d_rows)) return rc;
  if (!s->cyl) return PANO_OK;
  const int r0 = st * s->rows, r1 = std::min(s->oh, r0 + s->rows);
  return persp_correct_rows(s->st.ctx, s->d_band, row0, s->corr, s->ow, s->oh, &s->p, s->d_strip, r0, r1);
}

static int sweep_plan_out(int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                          const pano_params* p, int out_w, int out_h, const double* corr, int strip_rows,
                          const size_t* src_bytes, size_t keep_bytes, int* n_strips, int* band, unsigned char* reads,
                          unsigned char* uploads, unsigned char* kept, long long* n_uploads,
                          unsigned long long* upload_bytes, unsigned long long* retained_high) {
  if (!g) return PANO_ERR_INVALID;
  SweepPlan pl;
  if (int rc = make_plan(n, imgs, bands, p, out_w, out_h, strip_rows, src_bytes, keep_bytes, corr, &pl)) return rc;
  if (n_strips) *n_strips = pl.strips;
  if (band) std::copy(pl.band.begin(), pl.band.end(), band);
  if (reads) std::copy(pl.reads.begin(), pl.reads.end(), reads);
  if (uploads) std::copy(pl.uploads.begin(), pl.uploads.end(), uploads);
  if (kept) std::copy(pl.kept.begin(), pl.kept.end(), kept);
  if (n_uploads) *n_uploads = pl.n_uploads;
  if (upload_bytes) *upload_bytes = pl.upload_bytes;
  if (retained_high) *retained_high = pl.retained_high;
  return PANO_OK;
}

// The sweep of pano_blend_sweep_create (corr null) or pano_blend_sweep_create_cyl (ct: the sources' warps).
static int sweep_create(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                        const pano_params* p, int out_w, int out_h, const CylTabs* ct, const double* corr,
                        int strip_rows, const size_t* src_bytes, size_t keep_bytes, int crop, pano_blend_sweep** out) {
  std::unique_ptr<pano_blend_sweep> s(new pano_blend_sweep);
  s->st.ctx = ctx; s->n = n; s->bands = bands; s->ow = out_w; s->oh = out_h; s->rows = std::min(strip_rows, out_h);
  s->p = *p; s->g = *g;
  s->imgs.assign(imgs, imgs + n);
  s->cyl = ct != nullptr;
  s->src_w.resize(n); s->src_h.resize(n);
  for (int k = 0; k < n; ++k) {
    s->src_w[k] = ct ? ct->w[k] : imgs[k].w;
    s->src_h[k] = ct ? ct->h[k] : imgs[k].h;
  }
  std::vector<double> tab;
  int rc = blend_sweep_tables(ctx, n, imgs, g, bands, p, out_w, out_h, &tab);
  if (rc) return rc;
  s->bytes.resize(n);
  for (int k = 0; k < n; ++k) s->bytes[k] = src_bytes ? src_bytes[k] : (size_t)s->src_w[k] * s->src_h[k] * 3;
  if (make_plan(n, imgs, bands, p, out_w, out_h, strip_rows, s->bytes.data(), keep_bytes, corr, &s->plan))
    return ctx_fail(ctx, PANO_ERR_INVALID, "blend sweep: a source of 0 bytes");
  if (!tab.empty()) {
    if ((rc = s->d_tab.alloc(ctx, tab.size()))) return rc;
    if ((rc = ctx_put(ctx, s->d_tab, tab.data(), tab.size() * sizeof(double)))) return rc;
  }
  if (ct) {
    memcpy(s->corr, corr, sizeof(s->corr));
    s->ct = *ct;
    if ((rc = s->d_cyl_tab.alloc(ctx, std::max<size_t>(ct->tabs.size(), 1)))) return rc;
    if ((rc = ctx_put(ctx, s->d_cyl_tab, ct->tabs.data(), ct->tabs.size() * sizeof(double)))) return rc;
    int band_rows = 0;
    for (int st = 0; st < s->plan.strips; ++st)
      band_rows = std::max(band_rows, s->plan.band[2 * st + 1] - s->plan.band[2 * st]);
    if (band_rows > 0 && (rc = s->d_band.alloc(ctx, (size_t)band_rows * out_w * 3))) return rc;
  }
  if ((rc = s->d_strip.alloc(ctx, (size_t)s->rows * out_w * 3))) return rc;
  if ((rc = s->d_rgb.alloc(ctx, (size_t)out_w * out_h * 3))) return rc;
  if ((rc = s->d_rect.alloc(ctx, 4))) return rc;
  if (crop) {
    pano_crop_scan* c = nullptr;
    if ((rc = pano_crop_scan_create(ctx, out_w, out_h, &c))) return rc;
    s->scan.reset(c);
  }
  s->held.resize(n);
  *out = s.release();
  return PANO_OK;
}

extern "C" {

int pano_blend_sweep_plan(int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                          const pano_params* p, int out_w, int out_h, int strip_rows, const size_t* src_bytes,
                          size_t keep_bytes, int* n_strips, unsigned char* reads, unsigned char* uploads,
                          unsigned char* kept, long long* n_uploads, unsigned long long* upload_bytes,
                          unsigned long long* retained_high) {
  return sweep_plan_out(n, imgs, g, bands, p, out_w, out_h, nullptr, strip_rows, src_bytes, keep_bytes, n_strips,
                        nullptr, reads, uploads, kept, n_uploads, upload_bytes, retained_high);
}

int pano_blend_sweep_plan_cyl(int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                              const pano_params* p, int out_w, int out_h, const double corr_inv[9], int strip_rows,
                              const size_t* src_bytes, size_t keep_bytes, int* n_strips, int* band,
                              unsigned char* reads, unsigned char* uploads, unsigned char* kept, long long* n_uploads,
                              unsigned long long* upload_bytes, unsigned long long* retained_high) {
  if (!corr_inv) return PANO_ERR_INVALID;
  return sweep_plan_out(n, imgs, g, bands, p, out_w, out_h, corr_inv, strip_rows, src_bytes, keep_bytes, n_strips,
                        band, reads, uploads, kept, n_uploads, upload_bytes, retained_high);
}

int pano_blend_sweep_create(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g,
                            int bands, const pano_params* p, int out_w, int out_h, int strip_rows,
                            const size_t* src_bytes, size_t keep_bytes, int crop, pano_blend_sweep** out) {
  ctx_enter(ctx);
  if (!ctx || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  if (n <= 0 || !imgs || !g || !p || bands < 0 || strip_rows < 1) return ctx_fail(ctx, PANO_ERR_INVALID, "blend sweep: bad argument");
  if (n > PANO_MAX_IMAGES) return ctx_fail(ctx, PANO_ERR_INVALID, "blend sweep: %d images (limit %d)", n, PANO_MAX_IMAGES);
  return sweep_create(ctx, n, imgs, g, bands, p, out_w, out_h, nullptr, nullptr, strip_rows, src_bytes, keep_bytes,
                      crop, out);
}

int pano_blend_sweep_create_cyl(pano_ctx* ctx, int n, const pano_blend_image* imgs, const int* src_w,
                                const int* src_h, double h_factor, const pano_blend_geom* g, int bands,
                                const pano_params* p, int out_w, int out_h, const double corr_inv[9], int strip_rows,
                                const size_t* src_bytes, size_t keep_bytes, int crop, pano_blend_sweep** out) {
  ctx_enter(ctx);
  if (!ctx || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  if (n <= 0 || !imgs || !g || !p || !corr_inv || bands < 0 || strip_rows < 1)
    return ctx_fail(ctx, PANO_ERR_INVALID, "cylinder blend sweep: bad argument");
  CylTabs ct;
  if (int rc = cyl_tabs(ctx, n, imgs, src_w, src_h, h_factor, p, &ct)) return rc;
  return sweep_create(ctx, n, imgs, g, bands, p, out_w, out_h, &ct, corr_inv, strip_rows, src_bytes, keep_bytes, crop,
                      out);
}

int pano_blend_sweep_next(pano_blend_sweep* s, unsigned char* want) {
  if (!s) return PANO_ERR_INVALID;
  ctx_enter(s->st.ctx);
  if (s->st.err) return s->st.err;
  const bool over = s->done >= s->plan.strips;
  if (want)
    for (int k = 0; k < s->n; ++k) want[k] = over ? 0 : s->plan.uploads[(size_t)s->done * s->n + k];
  return over ? -1 : s->done;
}

int pano_blend_sweep_strip(pano_blend_sweep* s, const void* const* srcs, const int* formats, int kind) {
  if (!s) return PANO_ERR_INVALID;
  Sticky& ss = s->st;
  pano_ctx* ctx = ss.ctx;
  ctx_enter(ctx);
  if (ss.err) return ss.err;
  if (ss.finished || s->done >= s->plan.strips) return ss.misuse("blend sweep: strip after the last");
  if (!srcs) return ss.misuse("blend sweep: null source list");
  SrcKind sk;
  if (int rc = src_kind(ctx, "blend sweep", kind, &sk)) return ss.fail(rc);
  const bool u8 = sk.u8;
  if (u8 && !formats) return ss.misuse("blend sweep: null format list");
  const int n = s->n, st = s->done;
  const unsigned char* up = &s->plan.uploads[(size_t)st * n];
  std::vector<int> fmt(n, 3);
  std::vector<size_t> sz(n, 0);
  std::vector<int> list;           // the images handed over, in order
  for (int k = 0; k < n; ++k) {
    if (!srcs[k] && up[k]) return ss.misuse("blend sweep: strip %d needs image %d", st, k);
    if (srcs[k] && !up[k]) return ss.misuse("blend sweep: strip %d was not to be given image %d", st, k);
    if (!srcs[k]) continue;
    fmt[k] = u8 ? formats[k] : 3;
    if (int rc = src_check(ctx, "blend sweep", sk, k, fmt[k], srcs[k])) return ss.fail(rc);
    sz[k] = src_bytes(s->src_w[k], s->src_h[k], u8, fmt[k]);
    if (sz[k] > s->bytes[k])
      return ss.misuse("blend sweep: image %d takes %zu bytes, planned with %zu", k, sz[k], s->bytes[k]);
    list.push_back(k);
  }
  if (int rc = sweep_wait_previous(s)) return rc;
  if (int rc = sweep_blend(s, st, srcs, u8, sk.host, fmt, sz)) return ss.fail(rc);
  const int row0 = st * s->rows, row1 = std::min(s->oh, row0 + s->rows);
  if (s->scan)
    if (int rc = pano_crop_scan_add_dev(s->scan.get(), s->d_strip, row1 - row0)) return ss.fail(rc);
  if (int rc = pano_mat32f_to_rgb8_dev(ctx, s->d_strip, s->ow, row1 - row0, nullptr, s->d_rgb + (size_t)row0 * s->ow * 3))
    return ss.fail(rc);
  // drop what the plan does not keep past this strip (freed in stream order, after its readers)
  unsigned long long kept_bytes = 0;
  const unsigned char* hold = &s->plan.held[(size_t)st * n];
  for (int k = 0; k < n; ++k) {
    if (!hold[k]) s->held[k] = Held();
    else kept_bytes += s->bytes[k];
  }
  s->uploads += (long long)list.size();
  for (int k : list) s->upload_bytes += s->bytes[k];
  s->retained_high = std::max(s->retained_high, kept_bytes);
  ++s->done;
  return PANO_OK;
}

int pano_blend_sweep_finish_dev(pano_blend_sweep* s, int out_format, unsigned char* d_out, int rect[4]) {
  if (!s) return PANO_ERR_INVALID;
  Sticky& ss = s->st;
  pano_ctx* ctx = ss.ctx;
  ctx_enter(ctx);
  if (ss.err) return ss.err;
  if (!d_out || !rect) return ss.misuse("blend sweep: null output");
  if (ss.finished) return ss.misuse("blend sweep: already finished");
  if (s->done < s->plan.strips) return ss.misuse("blend sweep: finish after %d of %d strips", s->done, s->plan.strips);
  if (out_format != PANO_PIX_RGB && out_format != PANO_PIX_RGBA && out_format != PANO_PIX_RGB_PLANAR)
    return ss.misuse("blend sweep: output format %#x", out_format);
  ss.finished = true;
  if (int rc = sweep_wait_previous(s)) return rc;
  int r[4] = {0, 0, s->ow, s->oh};
  if (s->scan)
    if (int rc = pano_crop_scan_rect(s->scan.get(), r)) return ss.fail(rc);
  if (int rc = ctx_put(ctx, s->d_rect, r, sizeof(r))) return ss.fail(rc);
  if (int rc = pano_rgb8_crop_to_pix8_dev(ctx, s->d_rgb, s->ow, s->oh, s->d_rect, out_format, d_out))
    return ss.fail(rc);
  for (int q = 0; q < 4; ++q) rect[q] = r[q];
  return PANO_OK;
}

int pano_blend_sweep_stats(const pano_blend_sweep* s, long long* uploads, unsigned long long* upload_bytes,
                           unsigned long long* retained_high) {
  if (!s) return PANO_ERR_INVALID;
  if (uploads) *uploads = s->uploads;
  if (upload_bytes) *upload_bytes = s->upload_bytes;
  if (retained_high) *retained_high = s->retained_high;
  return PANO_OK;
}

void pano_blend_sweep_free(pano_blend_sweep* s) {
  if (s) ctx_enter(s->st.ctx);
  delete s;
}

}  // extern "C"
