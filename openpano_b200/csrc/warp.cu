// warp.cu — cylindrical pre-warp of an image and its keypoints.
//
// Replaces CylinderWarper::warp (stitch/warp.hh:41-66) = CylinderProject::project
// (stitch/warp.cc:25-67), proj/proj_r (:13-23), get_projector (:70-75).
// All geometry is f64.  The transcendental part of the inverse map depends only
// on the destination COLUMN (x = r*tan(px)+cx, 1/cos(px)), so it is evaluated on
// the host with the same libm the reference calls and uploaded as two per-column
// tables; the kernel then performs only IEEE mul/div/add and the f32 bilinear
// gather, which makes the image bit-identical to the reference.
#include "common.cuh"
#include <math.h>
#include <float.h>
#include <string.h>
#include <vector>
#include <algorithm>

struct CylProj { double cx, cy; int r; int sizefactor; };

static CylProj get_projector(int w, int h, double h_factor, const pano_params* p) {
  CylProj c;
  c.r = (int)(hypot((double)w, (double)h) * (p->focal_length / 43.266));
  c.cx = w / 2;
  c.cy = h / 2 * h_factor;
  c.sizefactor = c.r;
  return c;
}

static void proj(const CylProj& c, double px, double py, double* ox, double* oy) {
  *ox = atan((px - c.cx) / c.r);
  *oy = (py - c.cy) / hypot(px - c.cx, (double)c.r);
}

// Bounds of proj over the whole pixel grid (warp.cc:47-52 scans every pixel; min
// starts at +max, max starts at 0).  proj.x is monotone in the column and proj.y,
// for a fixed row, is extremal at the column nearest the centre, so the scan
// reduces to the border rows/columns — evaluated with the same expressions.
static void proj_bounds(const CylProj& c, int w, int h, double* minx, double* miny, double* maxx, double* maxy) {
  double mnx = DBL_MAX, mny = DBL_MAX, mxx = 0, mxy = 0;
  const int rows[2] = {0, h - 1};
  for (int ri = 0; ri < 2; ++ri)
    for (int j = 0; j < w; ++j) {
      double x, y;
      proj(c, j, rows[ri], &x, &y);
      if (x < mnx) mnx = x;
      if (y < mny) mny = y;
      if (mxx < x) mxx = x;
      if (mxy < y) mxy = y;
    }
  const int cols[2] = {0, w - 1};
  for (int ci = 0; ci < 2; ++ci)
    for (int i = 0; i < h; ++i) {
      double x, y;
      proj(c, cols[ci], i, &x, &y);
      if (x < mnx) mnx = x;
      if (y < mny) mny = y;
      if (mxx < x) mxx = x;
      if (mxy < y) mxy = y;
    }
  *minx = mnx; *miny = mny; *maxx = mxx; *maxy = mxy;
}

// warp.cc:46-67 project(Shape2D&, pts)
static void project_shape(const CylProj& c, int* w, int* h, double* kpts, int nk, double* offx, double* offy) {
  double minx, miny, maxx, maxy;
  proj_bounds(c, *w, *h, &minx, &miny, &maxx, &maxy);
  maxx = maxx * c.sizefactor; maxy = maxy * c.sizefactor;
  minx = minx * c.sizefactor; miny = miny * c.sizefactor;
  double rsx = maxx - minx, rsy = maxy - miny;
  *offx = minx * (-1); *offy = miny * (-1);
  int sx = (int)rsx, sy = (int)rsy;
  for (int i = 0; i < nk; ++i) {
    double x, y;
    proj(c, kpts[2 * i] + *w / 2, kpts[2 * i + 1] + *h / 2, &x, &y);
    x = x * c.sizefactor + *offx;
    y = y * c.sizefactor + *offy;
    x -= sx / 2;
    y -= sy / 2;
    kpts[2 * i] = x; kpts[2 * i + 1] = y;
  }
  *w = sx; *h = sy;
}

bool cyl_map(int w, int h, double h_factor, const pano_params* p, double* kpts, int nk, CylMap* m,
             std::vector<double>* tabs) {
  CylProj c = get_projector(w, h, h_factor, p);
  if (c.r <= 0) return false;
  int sw = w, sh = h;
  double offx, offy;
  project_shape(c, &sw, &sh, kpts, nk, &offx, &offy);
  m->ow = sw; m->oh = sh;
  m->r = (double)c.r; m->cy = c.cy; m->offy = offy; m->sizefactor_inv = 1.0 / c.sizefactor;
  if (sw <= 0 || sh <= 0) return true;
  const size_t t0 = tabs->size();
  tabs->resize(t0 + 2 * (size_t)sw);
  for (int j = 0; j < sw; ++j) {                                            // warp.cc:19-23 proj_r per column
    double px = ((double)j - offx) * m->sizefactor_inv;
    (*tabs)[t0 + j] = c.r * tan(px) + c.cx;
    (*tabs)[t0 + sw + j] = cos(px);
  }
  return true;
}

// one thread per destination pixel (warp.cc:33-41)
__global__ void k_cyl_warp(const float* __restrict__ src, int w, int h, float* __restrict__ dst, int ow, int oh,
                           const double* __restrict__ col_x, const double* __restrict__ col_cos, double r,
                           double cy, double offy, double sizefactor_inv) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  int i = blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= ow || i >= oh) return;
  float o0, o1, o2;
  cyl_warp_px([&] { return SrcF32{src}; }, w, h, col_x, col_cos, r, cy, offy, sizefactor_inv, i, j, &o0, &o1, &o2);
  float* p = dst + ((size_t)i * ow + j) * 3;
  p[0] = o0; p[1] = o1; p[2] = o2;
}

// The same for a batch of device-resident images: blockIdx.z = image; per-image parameters and the
// two per-column tables (concatenated) sit in device memory.  Src is the batch's reader (src_reader); an 8-bit
// reader converts every tap as read_img converts it, so the warp of the pixels is the warp of read_img's f32 image.
struct CylJobDev {
  const void* src;              // h×w×3 f32 or 8-bit pixels in format `channels`
  float* dst;
  int w, h, ow, oh;
  int channels;                 // 8-bit sources only: the PANO_PIX_* format
  long long tab_off;            // first entry of this image's col_x[ow] followed by col_cos[ow]
  double r, cy, offy, sizefactor_inv;
};

template <class Src>
__global__ void k_cyl_warp_batch(const CylJobDev* __restrict__ jobs, const double* __restrict__ tabs) {
  __shared__ float lut[Src::kLut ? 256 : 1];
  if constexpr (Src::kLut) {      // every thread of the 256 takes part, before any leaves at the edge below
    build_rgb8_lut(lut, threadIdx.y * blockDim.x + threadIdx.x);
    __syncthreads();
  }
  const CylJobDev jb = jobs[blockIdx.z];
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  int i = blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= jb.ow || i >= jb.oh) return;
  const double* col_x = tabs + jb.tab_off;
  float o0, o1, o2;
  cyl_warp_px([&] { return Src::at(jb.src, jb.w, jb.h, jb.channels, lut); }, jb.w, jb.h, col_x, col_x + jb.ow, jb.r, jb.cy, jb.offy,
              jb.sizefactor_inv, i, j, &o0, &o1, &o2);
  float* p = jb.dst + ((size_t)i * jb.ow + j) * 3;
  p[0] = o0; p[1] = o1; p[2] = o2;
}

// Both batch entry points.  pix / channels: 8-bit device sources (jobs[k].d_rgb_hwc ignored), else null
// and jobs[k].d_rgb_hwc are the sources.  The keypoints and the per-column tables are host arithmetic on
// the shapes alone, the same for both.
static int cyl_warp_batch(pano_ctx* ctx, int n, const pano_cyl_job* jobs, double h_factor, const pano_params* p,
                          const unsigned char* const* pix = nullptr, const int* channels = nullptr) {
  if (!ctx || n < 0 || (n && !jobs) || !p) return PANO_ERR_INVALID;
  if (n > PANO_MAX_IMAGES)   // images on gridDim.z
    return ctx_fail(ctx, PANO_ERR_INVALID, "cyl warp: %d images in one batch (limit %d): split the batch", n, PANO_MAX_IMAGES);
  if (n == 0) return PANO_OK;
  std::vector<CylJobDev> dj(n);
  std::vector<double> tabs;
  int max_ow = 0, max_oh = 0;
  for (int k = 0; k < n; ++k) {
    const pano_cyl_job& jb = jobs[k];
    if ((!pix && !jb.d_rgb_hwc) || !jb.d_out_hwc || jb.w <= 1 || jb.h <= 1 || jb.n_kpts < 0 || (jb.n_kpts && !jb.kpts_xy))
      return ctx_fail(ctx, PANO_ERR_INVALID, "cyl_warp_batch: job %d has a null pointer or an empty image", k);
    if (pix && !pix[k]) return ctx_fail(ctx, PANO_ERR_INVALID, "cyl_warp_batch rgb8: job %d has no pixels", k);
    if (pix)
      if (int rc = pix8_check(ctx, "cyl_warp_batch rgb8", k, channels[k], pix[k])) return rc;
    const size_t t0 = tabs.size();
    CylMap m;
    if (!cyl_map(jb.w, jb.h, h_factor, p, jb.kpts_xy, jb.n_kpts, &m, &tabs))   // keypoints: host arithmetic, in place
      return ctx_fail(ctx, PANO_ERR_INVALID, "cylinder radius <= 0");
    const int sw = m.ow, sh = m.oh;
    if (sw != jb.out_w || sh != jb.out_h || sw <= 0 || sh <= 0)
      return ctx_fail(ctx, PANO_ERR_INVALID, "cyl_warp_batch: job %d output buffer is %dx%d but the warp is %dx%d", k,
                      jb.out_w, jb.out_h, sw, sh);
    CylJobDev& d = dj[k];
    memset(&d, 0, sizeof(d));
    d.src = pix ? (const void*)pix[k] : jb.d_rgb_hwc;
    d.channels = pix ? channels[k] : 3;
    d.dst = jb.d_out_hwc;
    d.w = jb.w; d.h = jb.h; d.ow = sw; d.oh = sh;
    d.tab_off = (long long)t0;
    d.r = m.r; d.cy = m.cy; d.offy = m.offy; d.sizefactor_inv = m.sizefactor_inv;
    max_ow = std::max(max_ow, sw); max_oh = std::max(max_oh, sh);
  }
  DevBuf<CylJobDev> d_jobs;
  DevBuf<double> d_tabs;
  int rc = 0;
  if ((rc = d_jobs.alloc(ctx, dj.size())) || (rc = d_tabs.alloc(ctx, tabs.size()))) return rc;
  if ((rc = ctx_put(ctx, d_jobs, dj.data(), dj.size() * sizeof(CylJobDev)))) return rc;
  if ((rc = ctx_put(ctx, d_tabs, tabs.data(), tabs.size() * sizeof(double)))) return rc;
  dim3 b(32, 8), g(ceil_div(max_ow, 32), ceil_div(max_oh, 8), n);   // 256 threads: the 8-bit conversion table
  return with_reader(src_reader(pix ? channels : nullptr, n), [&](auto tag) -> int {
    using Src = typename decltype(tag)::type;
    PANO_LAUNCH(ctx, src_name<Src>(SRC_NAMES("k_cyl_warp")), k_cyl_warp_batch<Src>, g, b, 0, d_jobs, d_tabs);
    return PANO_OK;   // stream-ordered: the blocks are released after the kernel
  });
}

extern "C" {

int pano_cyl_warp_batch_dev(pano_ctx* ctx, int n, const pano_cyl_job* jobs, double h_factor, const pano_params* p) {
  ctx_enter(ctx);
  return cyl_warp_batch(ctx, n, jobs, h_factor, p);
}

int pano_cyl_warp_batch_rgb8_dev(pano_ctx* ctx, int n, const pano_cyl_job* jobs, const unsigned char* const* d_pix,
                                 const int* channels, double h_factor, const pano_params* p) {
  ctx_enter(ctx);
  if (!ctx) return PANO_ERR_INVALID;
  if (n > 0 && (!d_pix || !channels)) return ctx_fail(ctx, PANO_ERR_INVALID, "cyl_warp_batch rgb8: null source list");
  return cyl_warp_batch(ctx, n, jobs, h_factor, p, d_pix, channels);
}

int pano_cyl_warp_shape(int w, int h, double h_factor, const pano_params* p, int* ow, int* oh, double* offx,
                        double* offy) {
  if (w <= 0 || h <= 0 || !p || !ow || !oh || !offx || !offy) return PANO_ERR_INVALID;
  CylProj c = get_projector(w, h, h_factor, p);
  if (c.r <= 0) return PANO_ERR_INVALID;
  *ow = w; *oh = h;
  project_shape(c, ow, oh, nullptr, 0, offx, offy);
  return PANO_OK;
}

int pano_cyl_warp(pano_ctx* ctx, const float* rgb, int w, int h, double h_factor, const pano_params* p, float* out,
                  int ow, int oh, double* kpts, int nk) {
  ctx_enter(ctx);
  if (!ctx || !rgb || !out || !p || w <= 1 || h <= 1 || nk < 0 || (nk && !kpts)) return PANO_ERR_INVALID;
  CylMap m;
  std::vector<double> tab;   // per-column tables
  if (!cyl_map(w, h, h_factor, p, kpts, nk, &m, &tab)) return ctx_fail(ctx, PANO_ERR_INVALID, "cylinder radius <= 0");
  if (m.ow != ow || m.oh != oh || ow <= 0 || oh <= 0)
    return ctx_fail(ctx, PANO_ERR_INVALID, "cyl_warp: output buffer is %dx%d but the warp is %dx%d", ow, oh, m.ow,
                    m.oh);
  DevBuf<float> d_src, d_dst;
  DevBuf<double> d_tab;
  size_t bs = (size_t)w * h * 3 * sizeof(float), bd = (size_t)ow * oh * 3 * sizeof(float);
  int rc = 0;
  if ((rc = d_src.alloc(ctx, (size_t)w * h * 3)) || (rc = d_dst.alloc(ctx, (size_t)ow * oh * 3)) ||
      (rc = d_tab.alloc(ctx, tab.size())))
    return rc;
  PANO_CUDA(ctx, cudaMemcpyAsync(d_src, rgb, bs, cudaMemcpyHostToDevice, ctx->stream));
  PANO_CUDA(ctx, cudaMemcpyAsync(d_tab, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  dim3 b(32, 8), g(ceil_div(ow, 32), ceil_div(oh, 8));
  PANO_LAUNCH(ctx, "k_cyl_warp", k_cyl_warp, g, b, 0, d_src, w, h, d_dst, ow, oh, d_tab, d_tab + ow, m.r, m.cy, m.offy,
              m.sizefactor_inv);
  PANO_CUDA(ctx, cudaMemcpyAsync(out, d_dst, bd, cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PANO_OK;
}

}  // extern "C"
