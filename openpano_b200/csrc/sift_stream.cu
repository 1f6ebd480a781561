// sift_stream.cu — pano_sift_stream: SIFT fed window by window, LAZY_READ's feature stage
// (config.cfg:10-11, stitcherbase.cc:9-27).  Each window is one sift_run_batch over device pointers;
// host windows arrive through the upload ring (common.cuh), so window k+1's upload runs while window k's
// SIFT does.  A window's counts are read when the next window arrives (or at finish): a list overflow
// runs the window again with doubled lists while its sources are still resident (featureset_sync_counts),
// then its rows are packed into a block of their own and its lists go back to the pool.  finish gathers
// the packed blocks into one ordinary featureset.
#include "sift.cuh"
#include <algorithm>

namespace {

// Rows an image takes in a packed block: its count rounded up to 32, as pano_featureset_upload lays rows out.
long long packed_rows(int count) { return (count + 31LL) / 32 * 32; }

// The window that was queued last and whose counts have not been read yet.
struct PendingWindow {
  int first = 0, count = 0;
  int slot = -1;                          // ring slot of host sources, -1 for device sources
  std::unique_ptr<pano_featureset> fs;    // its lists at the context's capacity, and what a re-run needs
};

// A finished window: descriptors (rows × 128 f32), then coordinates (rows × 2 f64) followed by real
// coordinates (rows × 2 f64), each image's rows packed_rows(count) apart.
struct PackedWindow {
  long long rows = 0;
  DevBuf<float> desc;
  DevBuf<double> coor;
};

}  // namespace

struct pano_sift_stream {
  ~pano_sift_stream() {
    // the count read-back of a window never resolved still writes into its pinned block
    if (pending.fs && pending.fs->counts_pending) ctx_wait_signal(st.ctx, pending.fs->counts_token);
  }
  Sticky st;
  int n = 0, added = 0;
  std::vector<int> w, h;
  pano_params p;
  std::vector<int> count;                 // descriptors per image of the finished windows
  std::vector<PackedWindow> packed;
  UploadRing ring;
  PendingWindow pending;
};

// Reads the pending window's counts (a list overflow re-runs it), frees its ring slot and packs its rows.
static int sift_stream_resolve(pano_sift_stream* s) {
  PendingWindow& win = s->pending;
  if (!win.fs) return PANO_OK;
  pano_ctx* ctx = s->st.ctx;
  pano_featureset* fs = win.fs.get();
  if (int rc = featureset_sync_counts(fs)) return rc;
  if (win.slot >= 0) PANO_CUDA(ctx, s->ring.release(ctx, win.slot));   // its last reader is queued
  PackedWindow pw;
  std::vector<long long> off(win.count);
  for (int k = 0; k < win.count; ++k) {
    off[k] = pw.rows;
    pw.rows += packed_rows(fs->h_count[k]);
    s->count[win.first + k] = fs->h_count[k];
  }
  const size_t rows = (size_t)std::max(pw.rows, 1LL);
  if (int rc = pw.desc.alloc(ctx, rows * 128)) return rc;
  if (int rc = pw.coor.alloc(ctx, rows * 4)) return rc;
  std::vector<void*> dsts; std::vector<const void*> srcs; std::vector<size_t> sizes;
  for (int k = 0; k < win.count; ++k) {
    const size_t m = (size_t)fs->h_count[k];
    if (!m) continue;
    dsts.push_back(pw.desc + off[k] * 128); srcs.push_back(fs->d_desc + fs->base[k] * 128); sizes.push_back(m * 128 * sizeof(float));
    dsts.push_back(pw.coor + off[k] * 2); srcs.push_back(fs->d_coor + fs->base[k] * 2); sizes.push_back(m * 2 * sizeof(double));
    dsts.push_back(pw.coor + rows * 2 + off[k] * 2); srcs.push_back(fs->d_real + fs->base[k] * 2); sizes.push_back(m * 2 * sizeof(double));
  }
  if (int rc = ctx_copy_blocks(ctx, (int)dsts.size(), dsts.data(), srcs.data(), sizes.data())) return rc;
  win.fs.reset();   // the lists go back to the pool behind the copy
  s->packed.push_back(std::move(pw));
  return PANO_OK;
}

extern "C" {

int pano_sift_stream_create(pano_ctx* ctx, int n, const int* w, const int* h, const pano_params* p,
                            pano_sift_stream** out) {
  ctx_enter(ctx);
  if (!ctx || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  if (n <= 0 || !w || !h || !p) return ctx_fail(ctx, PANO_ERR_INVALID, "sift stream: bad argument");
  if (n > PANO_MAX_IMAGES) return ctx_fail(ctx, PANO_ERR_INVALID, "sift stream: %d images (limit %d)", n, PANO_MAX_IMAGES);
  for (int i = 0; i < n; ++i)
    if (w[i] < 2 || h[i] < 2) return ctx_fail(ctx, PANO_ERR_INVALID, "sift stream: image %d is %dx%d (at least 2x2)", i, w[i], h[i]);
  std::unique_ptr<pano_sift_stream> s(new pano_sift_stream);
  s->st.ctx = ctx; s->n = n; s->p = *p;
  s->w.assign(w, w + n); s->h.assign(h, h + n);
  s->count.assign(n, 0);
  *out = s.release();
  return PANO_OK;
}

int pano_sift_stream_add(pano_sift_stream* s, int first, int count, const void* const* srcs, int kind, int channels) {
  if (!s) return PANO_ERR_INVALID;
  pano_ctx* ctx = s->st.ctx;
  ctx_enter(ctx);
  SrcKind sk;
  if (int rc = s->st.add_check("sift stream", s->n, s->added, first, count, PANO_MAX_SIFT_BATCH, srcs, nullptr, kind,
                               channels, &sk))
    return rc;
  const bool u8 = sk.u8;

  std::vector<const void*> d_src(srcs, srcs + count);
  int slot = -1;
  if (sk.host) {   // queued on the copy stream first, so that it runs while the pending window's SIFT does
    std::vector<size_t> bytes(count);
    for (int k = 0; k < count; ++k)
      bytes[k] = src_bytes(s->w[first + k], s->h[first + k], u8, channels);
    if (int rc = s->ring.upload(ctx, "sift stream", count, srcs, bytes.data(), d_src.data(), &slot)) return s->st.fail(rc);
  }
  if (int rc = sift_stream_resolve(s)) return s->st.fail(rc);

  std::unique_ptr<pano_featureset> fs(new pano_featureset);
  fs->ctx = ctx;
  fs->src = d_src;
  fs->src_w.assign(s->w.begin() + first, s->w.begin() + first + count);
  fs->src_h.assign(s->h.begin() + first, s->h.begin() + first + count);
  fs->src_params = s->p;
  if (u8) fs->src_channels.assign(count, channels);
  int rc = sift_run_batch(ctx, count, d_src.data(), u8 ? fs->src_channels.data() : nullptr, fs->src_w.data(),
                          fs->src_h.data(), &s->p, fs.get(), nullptr, ctx_sift_cap(ctx));
  if (rc) return s->st.fail(rc);
  s->pending.first = first; s->pending.count = count; s->pending.slot = slot;
  s->pending.fs = std::move(fs);
  s->added += count;
  return PANO_OK;
}

int pano_sift_stream_finish(pano_sift_stream* s, pano_featureset** out) {
  if (!s) return PANO_ERR_INVALID;
  pano_ctx* ctx = s->st.ctx;
  ctx_enter(ctx);
  if (out) *out = nullptr;
  if (int rc = s->st.finish_check("sift stream", out, s->added, s->n)) return rc;
  if (int rc = sift_stream_resolve(s)) return s->st.fail(rc);

  // the packed windows back to back: their concatenation is the featureset's layout
  std::unique_ptr<pano_featureset> fs(new pano_featureset);
  fs->ctx = ctx; fs->n_images = s->n;
  fs->base.resize(s->n);
  long long total = 0;
  for (int i = 0; i < s->n; ++i) { fs->base[i] = total; total += packed_rows(s->count[i]); }
  const size_t rows = (size_t)std::max(total, 1LL);
  int rc = fs->d_desc.alloc(ctx, rows * 128);
  if (!rc) rc = fs->d_coor.alloc(ctx, rows * 4);
  if (!rc) rc = fs->d_count.alloc(ctx, s->n);
  if (rc) return s->st.fail(rc);
  fs->d_real = fs->d_coor + rows * 2;
  std::vector<void*> dsts; std::vector<const void*> srcs; std::vector<size_t> sizes;
  long long at = 0;
  for (const PackedWindow& pw : s->packed) {
    if (pw.rows) {
      const size_t wrows = (size_t)std::max(pw.rows, 1LL);
      dsts.push_back(fs->d_desc + at * 128); srcs.push_back(pw.desc); sizes.push_back((size_t)pw.rows * 128 * sizeof(float));
      dsts.push_back(fs->d_coor + at * 2); srcs.push_back(pw.coor); sizes.push_back((size_t)pw.rows * 2 * sizeof(double));
      dsts.push_back(fs->d_real + at * 2); srcs.push_back(pw.coor + wrows * 2); sizes.push_back((size_t)pw.rows * 2 * sizeof(double));
    }
    at += pw.rows;
  }
  if ((rc = ctx_copy_blocks(ctx, (int)dsts.size(), dsts.data(), srcs.data(), sizes.data()))) return s->st.fail(rc);
  if ((rc = ctx_put(ctx, fs->d_count, s->count.data(), s->n * sizeof(int)))) return s->st.fail(rc);
  s->packed.clear();   // back to the pool behind the copy
  fs->h_count = s->count;
  fs->counts_on_host = true;
  *out = fs.release();
  return PANO_OK;
}

void pano_sift_stream_free(pano_sift_stream* s) {
  if (s) ctx_enter(s->st.ctx);
  delete s;
}

}  // extern "C"
