// blend.cu — final composite: LinearBlender and MultiBandBlender.
//
// Replaces BlenderBase::add_image/run (stitch/blender.hh:14-59) for
// LinearBlender::run (stitch/blender.cc:24-96) and MultiBandBlender::run
// (stitch/multiband.cc:19-151).  The per-image inverse map, an opaque
// std::function in the reference, is the closed form of
// stitch/stitcher_image.cc:142-151 + stitch/projection.hh:14-71: its only
// transcendental terms depend on the canvas column (sin/cos of c.x) or row
// (tan of c.y), so they are tabulated on the host with the reference's libm and
// the kernels do IEEE f64 arithmetic only -> bit-identical coordinates.
#include "common.cuh"
#include "blend_rows.cuh"
#include "blur_tile.cuh"
#include <math.h>
#include <string.h>
#include <vector>
#include <algorithm>
#include <climits>
#include <memory>

struct BlendImg {
  const void* src;        // device: h×w×3 f32 (SrcF32), 8-bit pixels in format `channels` (SrcRgb8 / SrcPix8),
                          // or the image's cylinder warp, a CylImg (SrcCyl: pano_blend_stream_create_cyl)
  int w, h;
  int x0, y0, x1, y1;
  double hi[9];
  // multiband: the ROI is kept as FOUR PLANES (r, g, b, weight) of rh x pitch floats — the
  // reference's WeightedPixel (multiband.hh:13-23) de-interleaved, so that the weight map, the
  // blur and the accumulation each touch only the bytes they use and rows start on 128-byte lines
  long long roi_off;      // first float of plane 0 in the level buffers
  long long plane;        // floats per plane (pitch * rh)
  long long mask_off;     // first byte of the validity mask (same pitch)
  int rw, rh, pitch;
  int channels;           // 8-bit sources only: the PANO_PIX_* format
};

struct BlendGeom {
  int projection;
  double res_x, res_y, min_x, min_y;
  const double* col_sin;  // [tw+1] cylindrical/spherical
  const double* col_cos;
  const double* row_tan;  // [th+1] spherical
};

// stitcher_image.cc:142-151
__device__ __forceinline__ void coor_func(const BlendImg& im, const BlendGeom& g, int tx, int ty, double* ox, double* oy) {
  double cx = (double)tx * g.res_x + g.min_x;
  double cy = (double)ty * g.res_y + g.min_y;
  double hx, hy, hz;
  if (g.projection == PANO_PROJ_FLAT) { hx = cx; hy = cy; hz = 1.0; }
  else if (g.projection == PANO_PROJ_CYLINDRICAL) { hx = g.col_sin[tx]; hy = cy; hz = g.col_cos[tx]; }
  else { hx = g.col_sin[tx]; hy = g.row_tan[ty]; hz = g.col_cos[tx]; }
  double rx = im.hi[0] * hx + im.hi[1] * hy + im.hi[2] * hz;
  double ry = im.hi[3] * hx + im.hi[4] * hy + im.hi[5] * hz;
  double rz = im.hi[6] * hx + im.hi[7] * hy + im.hi[8] * hz;
  if (rz < 0) { *ox = -10; *oy = -10; return; }
  double denom = 1.0 / rz;
  *ox = rx * denom + im.w * 0.5;
  *oy = ry * denom + im.h * 0.5;
}

// ------------------------------------------------------------ per-tile image list
// Canvas kernels run one thread per output pixel over a 32x8 tile.  A pixel is covered
// by a few images, a mosaic has dozens: the first warp tests every image's range
// against the tile once and compacts the hits IN ORDER (the per-pixel loops must keep
// the reference's image order), so that the per-pixel loop runs over ~3 entries
// instead of n.  More than TILE_LIST_CAP hits: the pixel loop falls back to all n.
#define TILE_LIST_CAP 64
struct TileList { int n; unsigned short idx[TILE_LIST_CAP]; };

__device__ __forceinline__ void build_tile_list(const BlendImg* __restrict__ imgs, int n, int j0, int i0, int j1, int i1,
                                                TileList* tl) {
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  if (tid < 32) {
    int cnt = 0;
    for (int base = 0; base < n; base += 32) {
      const int k = base + tid;
      bool hit = false;
      if (k < n) {
        const BlendImg& im = imgs[k];
        hit = im.y0 <= i1 && im.y1 >= i0 && im.x0 <= j1 && im.x1 >= j0;   // inclusive: superset of both range rules
      }
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      if (hit) {
        const int slot = cnt + __popc(bal & ((1u << tid) - 1));
        if (slot < TILE_LIST_CAP) tl->idx[slot] = (unsigned short)k;
      }
      cnt += __popc(bal);
    }
    if (tid == 0) tl->n = (cnt <= TILE_LIST_CAP && n <= 65535) ? cnt : -1;
  }
  __syncthreads();
}

// ============================================================ linear blend
// blender.cc:24-96.  lazy != 0 selects the LAZY_READ branch (exclusive max
// bounds, accumulate then divide); otherwise the per-pixel branch.  Both add c·w and w
// of every covering image in image order, starting from 0.

// Adds the contributions of imgs[0, n) (tile list tl) at canvas pixel (i, j) to the sums.
template <class Src>
__device__ __forceinline__ void linear_add_px(const BlendImg* __restrict__ imgs, int n, const TileList& tl,
                                              const BlendGeom& g, int lazy, int ordered, const float* lut, int i, int j,
                                              float& s0, float& s1, float& s2, float& wsum) {
  const int nl = tl.n < 0 ? n : tl.n;
  for (int q = 0; q < nl; ++q) {
    const BlendImg& im = imgs[tl.n < 0 ? q : (int)tl.idx[q]];
    bool in = lazy ? (i >= im.y0 && i < im.y1 && j >= im.x0 && j < im.x1)
                   : (i >= im.y0 && i <= im.y1 && j >= im.x0 && j <= im.x1);
    if (!in) continue;
    double x, y;
    coor_func(im, g, j, i, &x, &y);
    if (x < 0 || x >= im.w || y < 0 || y >= im.h) continue;       // map_coor -> NaN
    float r = (float)y, c = (float)x;
    float c0, c1, c2;
    if (!interpolate_rgb(Src::at(im.src, im.w, im.h, im.channels, lut), im.w, im.h, r, c, &c0, &c1, &c2)) continue;
    if (c0 < 0) continue;
    float w = (float)(0.5 - fabs((double)(c / (float)im.w) - 0.5));
    if (!ordered) w = (float)((double)w * (0.5 - fabs((double)(r / (float)im.h) - 0.5)));
    s0 += c0 * w; s1 += c1 * w; s2 += c2 * w;
    wsum += w;
  }
}

// The final step of both branches: blender.cc:66-76 (lazy) and :91-92, -1 where nothing was added.
__device__ __forceinline__ void linear_resolve_px(int lazy, float s0, float s1, float s2, float wsum, float* p) {
  if (lazy) {
    if (wsum != 0.f) { p[0] = s0 / wsum; p[1] = s1 / wsum; p[2] = s2 / wsum; }
    else { p[0] = -1.f; p[1] = -1.f; p[2] = -1.f; }
  } else {
    if (wsum > 0) {
      float inv = (float)(1.0 / (double)wsum);
      p[0] = s0 * inv; p[1] = s1 * inv; p[2] = s2 * inv;
    } else { p[0] = -1.f; p[1] = -1.f; p[2] = -1.f; }
  }
}

template <class Src>
__global__ void k_linear_blend(const BlendImg* __restrict__ imgs, int n, BlendGeom g, int lazy, int ordered,
                               float* __restrict__ out, int tw, int row0, int row1) {
  // rows [row0, row1) of the canvas; `out` starts at row0 (a strip of a row-sharded mosaic, or the whole)
  __shared__ TileList tl;
  __shared__ float lut[Src::kLut ? 256 : 1];
  if constexpr (Src::kLut) build_rgb8_lut(lut, threadIdx.y * blockDim.x + threadIdx.x);   // ordered by the list's barrier
  {
    const int tj0 = blockIdx.x * blockDim.x, ti0 = row0 + blockIdx.y * blockDim.y;
    build_tile_list(imgs, n, tj0, ti0, tj0 + blockDim.x - 1, ti0 + blockDim.y - 1, &tl);
  }
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  int i = row0 + blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= tw || i >= row1) return;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, wsum = 0.f;
  linear_add_px<Src>(imgs, n, tl, g, lazy, ordered, lut, i, j, s0, s1, s2, wsum);
  linear_resolve_px(lazy, s0, s1, s2, wsum, out + ((size_t)(i - row0) * tw + j) * 3);
}

// One window of a blend stream: adds imgs[0, n) into the persistent sums of the stream's rows
// (sum: tw×rows×3, wsum: tw×rows, both zero at the start; canvas row row0 is their first row), one
// thread per pixel of the window's bounding rectangle [rx0, rx1) × [ry0, ry1), which lies in those
// rows.  Windows run in image order, so every pixel sees the float additions of k_linear_blend in
// the same order.
template <class Src>
__global__ void k_linear_accumulate(const BlendImg* __restrict__ imgs, int n, BlendGeom g, int lazy, int ordered,
                                    float* __restrict__ sum, float* __restrict__ wsum, int tw, int row0, int rx0, int ry0,
                                    int rx1, int ry1) {
  __shared__ TileList tl;
  __shared__ float lut[Src::kLut ? 256 : 1];
  if constexpr (Src::kLut) build_rgb8_lut(lut, threadIdx.y * blockDim.x + threadIdx.x);   // ordered by the list's barrier
  const int tj0 = rx0 + blockIdx.x * blockDim.x, ti0 = ry0 + blockIdx.y * blockDim.y;
  build_tile_list(imgs, n, tj0, ti0, tj0 + blockDim.x - 1, ti0 + blockDim.y - 1, &tl);
  const int j = tj0 + threadIdx.x, i = ti0 + threadIdx.y;
  if (tl.n == 0 || j >= rx1 || i >= ry1) return;
  const size_t t = (size_t)(i - row0) * tw + j;
  float* p = sum + t * 3;
  float s0 = p[0], s1 = p[1], s2 = p[2], ws = wsum[t];
  linear_add_px<Src>(imgs, n, tl, g, lazy, ordered, lut, i, j, s0, s1, s2, ws);
  p[0] = s0; p[1] = s1; p[2] = s2;
  wsum[t] = ws;
}

// The stream's last step: k_linear_blend's tail on the sums.  out may be `sum` itself.
__global__ void k_linear_resolve(const float* sum, const float* __restrict__ wsum, float* out, size_t n_px, int lazy) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_px) return;
  const float* p = sum + t * 3;
  linear_resolve_px(lazy, p[0], p[1], p[2], wsum[t], out + t * 3);
}

// Cylinder mode's perspective correction (cylstitcher.cc:139-180): a LinearBlender of the one image, the w×h
// mosaic, over ROI (0, 0)–(w, h) with the map inv.trans2d(c) (homography.hh:60-76) — no centre shift, no z test.
// One thread per pixel of output rows [row0, row1); `out` starts at row0.  Every output pixel lies in the ROI under
// both range rules, so the pixel is linear_add_px's one-image case; the taps come from the mosaic rows the band
// reader holds, judged against the whole mosaic's w×h.
struct PerspMap { double d[9]; };

template <class Src>
__global__ void k_persp_correct(BandImg band, PerspMap m, int w, int h, int lazy, int ordered, float* __restrict__ out,
                                int row0, int row1) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = row0 + blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= w || i >= row1) return;
  const double cx = (double)j, cy = (double)i;
  const double rx = m.d[0] * cx + m.d[1] * cy + m.d[2] * 1.0;
  const double ry = m.d[3] * cx + m.d[4] * cy + m.d[5] * 1.0;
  const double rz = m.d[6] * cx + m.d[7] * cy + m.d[8] * 1.0;
  const double denom = 1.0 / rz;
  const double x = rx * denom, y = ry * denom;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, wsum = 0.f;
  if (!(x < 0 || x >= w || y < 0 || y >= h)) {                       // map_coor -> NaN
    const float r = (float)y, c = (float)x;
    float c0, c1, c2;
    if (interpolate_rgb(Src::at(&band, w, h, 3, nullptr), w, h, r, c, &c0, &c1, &c2) && !(c0 < 0)) {
      float wt = (float)(0.5 - fabs((double)(c / (float)w) - 0.5));
      if (!ordered) wt = (float)((double)wt * (0.5 - fabs((double)(r / (float)h) - 0.5)));
      s0 += c0 * wt; s1 += c1 * wt; s2 += c2 * wt;
      wsum += wt;
    }
  }
  linear_resolve_px(lazy, s0, s1, s2, wsum, out + ((size_t)(i - row0) * w + j) * 3);
}

int persp_correct_rows(pano_ctx* ctx, const float* d_band, int b0, const double inv[9], int w, int h,
                       const pano_params* p, float* d_out, int row0, int row1) {
  if (row0 >= row1) return PANO_OK;
  PerspMap m;
  memcpy(m.d, inv, sizeof(m.d));
  const BandImg band{d_band, b0};
  const dim3 b(32, 8), g(ceil_div(w, 32), ceil_div(row1 - row0, 8));
  PANO_LAUNCH(ctx, src_name<SrcBand>(SRC_NAMES("k_persp_correct")), k_persp_correct<SrcBand>, g, b, 0, band, m, w, h,
              p->lazy_read, p->ordered_input, d_out, row0, row1);
  return PANO_OK;
}

// ============================================================ multiband
// multiband.cc:19-57 create_first_level
// The first level of an image depends on that image only: a blend stream runs this once per
// window over the window's entries.
template <class Src>
__global__ void k_mb_first_level(const BlendImg* __restrict__ imgs, BlendGeom g, float* __restrict__ cur,
                                 unsigned char* __restrict__ mask) {
  __shared__ float lut[Src::kLut ? 256 : 1];
  if constexpr (Src::kLut) {
    build_rgb8_lut(lut, threadIdx.y * blockDim.x + threadIdx.x);
    __syncthreads();
  }
  const BlendImg& im = imgs[blockIdx.z];
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  int i = blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= im.rw || i >= im.rh) return;
  double x, y;
  coor_func(im, g, j + im.x0, i + im.y0, &x, &y);
  float c0, c1, c2;
  bool ok = interpolate_rgb(Src::at(im.src, im.w, im.h, im.channels, lut), im.w, im.h, (float)y, (float)x, &c0, &c1,
                            &c2);
  if (ok && fminf(c0, fminf(c1, c2)) < 0) ok = false;
  const size_t o = (size_t)i * im.pitch + j;
  float* p = cur + im.roi_off + o;
  float ww = 0.f;
  if (!ok) { c0 = 0.f; c1 = 0.f; c2 = 0.f; }
  else {
    double ox = x / im.w - 0.5, oy = y / im.h - 0.5;
    double wd = (0.5 - fabs(ox)) * (0.5 - fabs(oy));
    if (wd < 0.0) wd = 0.0;
    ww = (float)(wd + 1e-6);
  }
  p[0] = c0; p[im.plane] = c1; p[2 * im.plane] = c2; p[3 * im.plane] = ww;
  mask[im.mask_off + o] = ok ? 0 : 1;
}

// multiband.cc:125-143 update_weight_map (first image with the largest weight wins)
__global__ void k_mb_weight_argmax(const BlendImg* __restrict__ imgs, int n, float* __restrict__ cur, int tw,
                                   int row0, int row1) {
  __shared__ TileList tl;
  {
    const int tj0 = blockIdx.x * blockDim.x, ti0 = row0 + blockIdx.y * blockDim.y;
    build_tile_list(imgs, n, tj0, ti0, tj0 + blockDim.x - 1, ti0 + blockDim.y - 1, &tl);
  }
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  int i = row0 + blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= tw || i >= row1) return;
  const int nl = tl.n < 0 ? n : tl.n;
  // Two passes so that the weight loads of all covering images are in flight together: a
  // store into `cur` between two loads from it would order them (the compiler cannot prove the
  // planes disjoint), and the kernel then crawls through one DRAM round trip per image.
  // Every location is read and written by this thread only, so the read-only path is safe.
  float mx = 0.f;
  int best = -1;
  for (int q = 0; q < nl; ++q) {
    const BlendImg& im = imgs[tl.n < 0 ? q : (int)tl.idx[q]];
    if (i >= im.y0 && i <= im.y1 && j >= im.x0 && j <= im.x1) {
      const float w = __ldg(cur + im.roi_off + 3 * im.plane + (size_t)(i - im.y0) * im.pitch + (j - im.x0));
      if (w > mx) { mx = w; best = q; }
    }
  }
  for (int q = 0; q < nl; ++q) {
    const BlendImg& im = imgs[tl.n < 0 ? q : (int)tl.idx[q]];
    if (i >= im.y0 && i <= im.y1 && j >= im.x0 && j <= im.x1)
      cur[im.roi_off + 3 * im.plane + (size_t)(i - im.y0) * im.pitch + (j - im.x0)] = q == best ? 1.f : 0.f;
  }
}

// gaussian.hh:29-90 on WeightedPixel: every channel of the pixel goes through the same
// column-then-row passes, i.e. four independent scalar planes.
struct BlurTaps { int center; float taps[64]; };
struct MbPlane { long long off; int w, h, pitch, pad; };   // one (image, channel) plane of a level buffer

// Both passes of one blur level on 64x32 tiles of every plane (blur_tile.cuh), PERSISTENT CTAs:
// the tile + halo of the next work item is fetched by TMA into the other half of a double
// buffer while this one is computed.  TMA zero-fills outside the ROI where the reference's
// line buffers replicate the ROI edge (gaussian.hh:52-58,74-81): border tiles patch those cells
// from the staged in-range ones.
template <int C>
__global__ void __launch_bounds__(BT_THREADS, 4)
k_mb_blur_tma(const MbPlane* __restrict__ planes, const int2* __restrict__ span, int n_planes, int n_tiles,
              const TmaDesc* __restrict__ maps, float* __restrict__ dst, const __grid_constant__ BlurTaps bt) {
  extern __shared__ __align__(128) float smem[];
  __shared__ __align__(8) uint64_t s_bar[2];
  __shared__ BlurTile s_tile[2];                   // looked up once per tile by thread 0 (binary search)
  constexpr int RX = (C + 3) & ~3;                 // TMA box origin: 16-byte aligned columns
  constexpr int GW = BT_W + 2 * RX, GH = BT_H + 2 * C;
  constexpr int GSZ = (GH * GW + 31) & ~31;
  float* grey0 = smem;
  float* colbuf = smem + 2 * GSZ;
  float* outT = colbuf + BLUR_COLBUF_FLOATS(C);
  const int tid = threadIdx.x;
  constexpr uint32_t tile_bytes = (uint32_t)(GH * GW * sizeof(float));
  int t = blockIdx.x;
  if (tid == 0) {
    sbar_init(sm_u32(&s_bar[0]), 1);
    sbar_init(sm_u32(&s_bar[1]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (t < n_tiles) {
      const BlurTile tl = find_blur_tile(span, n_planes, t);
      s_tile[0] = tl;
      sbar_expect_tx(sm_u32(&s_bar[0]), tile_bytes);
      tma_load_2d(sm_u32(grey0), maps + tl.om, tl.tx * BT_W - RX, tl.ty * BT_H - C, sm_u32(&s_bar[0]));
    }
  }
  __syncthreads();
  for (int it = 0; t < n_tiles; t += gridDim.x, ++it) {
    const int b = it & 1;
    float* grey = grey0 + b * GSZ;
    const BlurTile tl = s_tile[b];
    const MbPlane pl = planes[tl.om];
    const int x0 = tl.tx * BT_W, y0 = tl.ty * BT_H;
    if (tid == 0 && t + (int)gridDim.x < n_tiles) {
      const BlurTile nx = find_blur_tile(span, n_planes, t + gridDim.x);
      s_tile[b ^ 1] = nx;      // read by everyone after the barrier that ends this iteration
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      sbar_expect_tx(sm_u32(&s_bar[b ^ 1]), tile_bytes);
      tma_load_2d(sm_u32(grey0 + (b ^ 1) * GSZ), maps + nx.om, nx.tx * BT_W - RX, nx.ty * BT_H - C, sm_u32(&s_bar[b ^ 1]));
    }
    sbar_wait(sm_u32(&s_bar[b]), (uint32_t)(it >> 1) & 1u);
    if (x0 - RX < 0 || y0 - C < 0 || x0 + BT_W + RX > pl.w || y0 + BT_H + C > pl.h) {   // uniform per CTA
      for (int i = tid; i < GH * GW; i += BT_THREADS) {
        const int yy = i / GW, xx = i - yy * GW;
        const int gy = y0 + yy - C, gx = x0 + xx - RX;
        const int cy = min(max(gy, 0), pl.h - 1), cx = min(max(gx, 0), pl.w - 1);
        if (cy != gy || cx != gx) grey[i] = grey[(cy - y0 + C) * GW + (cx - x0 + RX)];
      }
      __syncthreads();
    }
    blur_level<C>(grey, colbuf, outT, bt.taps, C, RX, GW, tid);
    const int tx = tid & (BT_W - 1), ty = tid / BT_W;   // 64 x 4
    const int gx = x0 + tx;
    float* out = dst + pl.off;
#pragma unroll
    for (int i = 0; i < BT_H / 4; ++i) {
      const int y = ty + 4 * i, gy = y0 + y;
      if (gx < pl.w && gy < pl.h) out[(size_t)gy * pl.pitch + gx] = outT[y * (BT_W + 1) + tx];
    }
    __syncthreads();   // colbuf / outT / this staging buffer are free for the next tiles
  }
}

// Any other window width (GAUSS_WINDOW_FACTOR != 6, more than 5 bands): one tile per CTA,
// clamped loads, taps looped from the table.
#define MB_TW 64
#define MB_TH 32
__global__ void __launch_bounds__(256)
k_mb_blur_generic(const MbPlane* __restrict__ planes, const int2* __restrict__ span, int n_planes,
                  const float* __restrict__ src, float* __restrict__ dst, const __grid_constant__ BlurTaps bt) {
  extern __shared__ float mb_smem[];
  const BlurTile tl = find_blur_tile(span, n_planes, blockIdx.x);
  const MbPlane pl = planes[tl.om];
  const int tx0 = tl.tx * MB_TW, ty0 = tl.ty * MB_TH;
  const int c = bt.center, kw = 2 * c + 1;
  const int SW = MB_TW + 2 * c, SH = MB_TH + 2 * c;
  float* tile = mb_smem;                 // [SH][SW]
  float* colres = mb_smem + SH * SW;     // [MB_TH][SW]
  const float* base = src + pl.off;
  const int tid = threadIdx.x;
  for (int idx = tid; idx < SH * SW; idx += 256) {
    const int r = idx / SW, q = idx - r * SW;
    const int y = min(max(ty0 - c + r, 0), pl.h - 1), x = min(max(tx0 - c + q, 0), pl.w - 1);
    tile[idx] = __ldg(base + (size_t)y * pl.pitch + x);
  }
  __syncthreads();
  for (int idx = tid; idx < MB_TH * SW; idx += 256) {
    const int i = idx / SW, q = idx - i * SW;
    float acc = 0.f;
    const float* col = tile + i * SW + q;
    for (int k = 0; k < kw; ++k) acc += col[k * SW] * bt.taps[k];
    colres[idx] = acc;
  }
  __syncthreads();
  for (int idx = tid; idx < MB_TH * MB_TW; idx += 256) {
    const int i = idx / MB_TW, j = idx - i * MB_TW;
    if (ty0 + i >= pl.h || tx0 + j >= pl.w) continue;
    float acc = 0.f;
    const float* row = colres + i * SW + j;
    for (int k = 0; k < kw; ++k) acc += row[k] * bt.taps[k];
    dst[pl.off + (size_t)(ty0 + i) * pl.pitch + tx0 + j] = acc;
  }
}

// multiband.cc:75-108 per-level accumulate (+ :113-121 clamp on the last level).  `first`: no
// level has touched the strip yet, so every pixel is written (value, or -1 = Color::NO) and
// no separate fill pass is needed.
__global__ void k_mb_accumulate(const BlendImg* __restrict__ imgs, int n, const float* __restrict__ cur,
                                const float* __restrict__ next, const unsigned char* __restrict__ mask,
                                int first, int is_last, float* __restrict__ out, unsigned char* __restrict__ tmask, int tw,
                                int row0, int row1) {
  // rows [row0, row1) of the canvas; out / tmask start at row0
  __shared__ TileList tl;
  {
    const int tj0 = blockIdx.x * blockDim.x, ti0 = row0 + blockIdx.y * blockDim.y;
    build_tile_list(imgs, n, tj0, ti0, tj0 + blockDim.x - 1, ti0 + blockDim.y - 1, &tl);
  }
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  int i = row0 + blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= tw || i >= row1) return;
  const int nl = tl.n < 0 ? n : tl.n;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, wsum = 0.f;
  for (int q = 0; q < nl; ++q) {
    const BlendImg& im = imgs[tl.n < 0 ? q : (int)tl.idx[q]];
    if (!(i >= im.y0 && i <= im.y1 && j >= im.x0 && j <= im.x1)) continue;
    const size_t o = (size_t)(i - im.y0) * im.pitch + (j - im.x0);
    // the weight plane decides: colours are fetched only where this image contributes
    const float w = __ldg(cur + im.roi_off + 3 * im.plane + o);
    if (w <= 0) continue;
    if (mask[im.mask_off + o]) continue;
    const float* pc = cur + im.roi_off + o;
    const float c0 = __ldg(pc), c1 = __ldg(pc + im.plane), c2 = __ldg(pc + 2 * im.plane);
    if (!is_last) {
      const float* pn = next + im.roi_off + o;
      const float n0 = __ldg(pn), n1 = __ldg(pn + im.plane), n2 = __ldg(pn + 2 * im.plane);
      s0 += (c0 - n0) * w; s1 += (c1 - n1) * w; s2 += (c2 - n2) * w;
    } else {
      s0 += c0 * w; s1 += c1 * w; s2 += c2 * w;
    }
    wsum += w;
  }
  size_t t = (size_t)(i - row0) * tw + j;
  float* p = out + t * 3;
  bool touched = first ? false : tmask[t] != 0;
  float v0 = -1.f, v1 = -1.f, v2 = -1.f;
  if (touched) { v0 = p[0]; v1 = p[1]; v2 = p[2]; }
  bool dirty = first != 0;
  if (!((double)wsum < 1e-6)) {
    s0 /= wsum; s1 /= wsum; s2 /= wsum;
    if (!touched) { v0 = s0; v1 = s1; v2 = s2; touched = true; }
    else { v0 += s0; v1 += s1; v2 += s2; }
    dirty = true;
  }
  if (is_last && touched) {
    v0 = v0 < 1.0f ? v0 : 1.0f; v0 = v0 > 0.f ? v0 : 0.f;
    v1 = v1 < 1.0f ? v1 : 1.0f; v1 = v1 > 0.f ? v1 : 0.f;
    v2 = v2 < 1.0f ? v2 : 1.0f; v2 = v2 > 0.f ? v2 : 0.f;
    dirty = true;
  }
  if (dirty) { p[0] = v0; p[1] = v1; p[2] = v2; }
  if (first || touched) tmask[t] = touched ? 1 : 0;
}

__global__ void k_fill(float* __restrict__ p, size_t n, float v) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// ------------------------------------------------------------------ host driver

// Everything a blend derives from its arguments on the host, before any device work.
struct BlendJob {
  std::vector<BlendImg> imgs;
  std::vector<int> src;       // the caller's index of each entry of imgs (images that reach no row are left out)
  BlendGeom g;
  int tw = 0, th = 0;
  long long roi_floats = 0;   // floats of one level buffer (4 planes per image)
  long long mask_bytes = 0;
  int max_rw = 0, max_rh = 0;
  std::vector<BlurTaps> level_taps;
  int halo = 0;               // summed half-widths of the level blurs
  bool strip = false;
  int clip0 = INT_MIN, clip1 = INT_MAX;
  std::vector<double> tab;    // sin / cos per canvas column, tan per row (non-flat projections)
  size_t ncol = 0, nrow = 0;
};

// The device state of one blend: image table, projection tables and, for multiband, the ROI level
// buffers, masks, target mask and blur tables.
struct BlendDev {
  DevBuf<BlendImg> d_imgs;
  DevBuf<double> d_tab;
  DevBuf<float> d_cur, d_next;
  DevBuf<unsigned char> d_mask, d_tmask;
  DevBuf<MbPlane> d_planes;
  DevBuf<int2> d_span;
  DevBuf<TmaDesc> d_maps;
  std::vector<int> centers;   // distinct TMA blur half-widths
  int n_planes = 0, n_tiles = 0;
  int wrow0 = 0, wrow1 = 0;   // rows the weight map is needed on
};

template <int C>
static cudaError_t launch_mb_blur_tma(pano_ctx* ctx, int grid, const MbPlane* planes, const int2* span, int n_planes,
                                      int n_tiles, const TmaDesc* maps, float* dst, const BlurTaps& bt) {
  constexpr int RX = (C + 3) & ~3, GW = BT_W + 2 * RX, GH = BT_H + 2 * C, GSZ = (GH * GW + 31) & ~31;
  const size_t smem = (size_t)(2 * GSZ + BLUR_COLBUF_FLOATS(C) + BT_H * (BT_W + 1)) * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(k_mb_blur_tma<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_mb_blur_tma<C><<<grid, BT_THREADS, smem, ctx->stream>>>(planes, span, n_planes, n_tiles, maps, dst, bt);
  return cudaGetLastError();
}

// Validates the images (need_src: every rgb_hwc must be set) and builds the job of rows [row0, row1).
// pix / channels (8-bit sources, else null): the images' pixels instead of rgb_hwc.
// The blur taps of every multiband level (multiband.cc:145-151); returns their summed half-widths, or -kw for
// a window wider than the tap table.
static int level_taps(int bands, int gauss_window_factor, std::vector<BlurTaps>* taps) {
  int halo = 0;
  for (int level = 0; level + 1 < bands; ++level) {
    float sigma = (float)(sqrt(level * 2 + 1.0) * 4);
    BlurTaps bt;
    memset(&bt, 0, sizeof(bt));
    int kw = host_gauss_kernel(sigma, gauss_window_factor, bt.taps, 63);
    if (kw < 0) return kw;
    bt.center = kw / 2;
    halo += bt.center;
    if (taps) taps->push_back(bt);
  }
  return halo;
}

int blend_halo(int bands, const pano_params* p) { return level_taps(bands, p->gauss_window_factor, nullptr); }

// Multiband on a row strip: a band at level l of pixel p depends on level 0 inside a
// radius of the summed half-widths of the blurs up to l, so the strip is computed from
// each image's ROI clipped to [row0 - H, row1 + H) with H = that sum over all blurred
// levels.  The replicate rule at a clipped edge differs from the true neighbourhood only
// within H rows of it, i.e. outside the strip; true ROI edges are kept as they are.
// [*clip0, *clip1]: the ROI rows kept (INT_MIN / INT_MAX where nothing is clipped).
static void strip_clip(int bands, int halo, int oh, int row0, int row1, int* clip0, int* clip1) {
  const bool strip = bands > 0 && (row0 != 0 || row1 != oh);
  *clip0 = (strip && row0 > 0) ? std::max(0, row0 - halo) : INT_MIN;
  *clip1 = (strip && row1 < oh) ? row1 + halo - 1 : INT_MAX;
}

bool blend_strip_reads(const pano_blend_image& im, int bands, int halo, int oh, int row0, int row1) {
  if (row0 == 0 && row1 == oh) return true;
  if (bands == 0) return im.y0 < row1 && im.y1 >= row0;
  int c0, c1;
  strip_clip(bands, halo, oh, row0, row1, &c0, &c1);
  return std::max(im.y0, c0) <= std::min(im.y1, c1);
}

static int blend_plan(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                      const pano_params* p, int ow, int oh, int row0, int row1, bool need_src, BlendJob* job,
                      const unsigned char* const* pix = nullptr, const int* channels = nullptr, bool tables = true) {
  job->halo = level_taps(bands, p->gauss_window_factor, &job->level_taps);
  if (job->halo < 0) return ctx_fail(ctx, PANO_ERR_INVALID, "blend: gaussian window %d too wide", -job->halo);
  job->strip = bands > 0 && (row0 != 0 || row1 != oh);
  strip_clip(bands, job->halo, oh, row0, row1, &job->clip0, &job->clip1);
  job->imgs.reserve(n);
  for (int k = 0; k < n; ++k) {
    const pano_blend_image& s = imgs[k];
    if ((need_src && !s.rgb_hwc) || s.w < 2 || s.h < 2 || s.x1 < s.x0 || s.y1 < s.y0 || s.x0 < 0 || s.y0 < 0)
      return ctx_fail(ctx, PANO_ERR_INVALID, "blend: image %d has an invalid shape or range", k);
    if (pix && !pix[k]) return ctx_fail(ctx, PANO_ERR_INVALID, "blend: image %d has no pixels", k);
    if (pix)
      if (int rc = pix8_check(ctx, "blend", k, channels[k], pix[k])) return rc;
    job->tw = std::max(job->tw, s.x1); job->th = std::max(job->th, s.y1);
    BlendImg d;
    memset(&d, 0, sizeof(d));
    d.src = pix ? (const void*)pix[k] : s.rgb_hwc;
    d.w = s.w; d.h = s.h;
    d.x0 = s.x0; d.x1 = s.x1;
    d.y0 = std::max(s.y0, job->clip0); d.y1 = std::min(s.y1, job->clip1);
    if (d.y0 > d.y1) continue;                         // no row of this image reaches the strip
    memcpy(d.hi, s.homo_inv, sizeof(d.hi));
    d.rw = d.x1 - d.x0 + 1; d.rh = d.y1 - d.y0 + 1;
    d.pitch = (int)align_up((size_t)d.rw, 32);
    d.plane = (long long)d.pitch * d.rh;
    d.roi_off = job->roi_floats;
    d.mask_off = job->mask_bytes;
    d.channels = pix ? channels[k] : 3;
    job->roi_floats += 4 * d.plane;
    job->mask_bytes += d.plane;
    job->max_rw = std::max(job->max_rw, d.rw); job->max_rh = std::max(job->max_rh, d.rh);
    job->imgs.push_back(d);
    job->src.push_back(k);
  }
  if (job->tw != ow || job->th != oh || ow <= 0 || oh <= 0)
    return ctx_fail(ctx, PANO_ERR_INVALID, "blend: output is %dx%d but target_size is %dx%d", ow, oh, job->tw, job->th);
  if (job->imgs.empty()) return PANO_OK;
  // ROIs reach one pixel past the canvas (inclusive max): tables cover [0, tw] / [0, th]
  job->ncol = (size_t)job->tw + 2; job->nrow = (size_t)job->th + 2;
  if (tables && g->projection != PANO_PROJ_FLAT) {
    job->tab.resize(2 * job->ncol + job->nrow);
    for (size_t j = 0; j < job->ncol; ++j) {
      double cx = (double)j * g->res_x + g->proj_min_x;
      job->tab[j] = sin(cx); job->tab[job->ncol + j] = cos(cx);
    }
    for (size_t i = 0; i < job->nrow; ++i) {
      double cy = (double)i * g->res_y + g->proj_min_y;
      job->tab[2 * job->ncol + i] = tan(cy);
    }
  }
  job->g.projection = g->projection; job->g.res_x = g->res_x; job->g.res_y = g->res_y;
  job->g.min_x = g->proj_min_x; job->g.min_y = g->proj_min_y;
  return PANO_OK;
}

// Allocates and uploads the device state of `job` (rows [row0, row1)).  shared_tab: the device projection
// tables of the same canvas and geometry, made once for many strips (job->tab is then empty), else null.
static int blend_dev_setup(pano_ctx* ctx, BlendJob* job, int bands, int row0, int row1, BlendDev* d,
                           const double* shared_tab = nullptr) {
  const int n = (int)job->imgs.size(), tw = job->tw, th = job->th;
  int rc = 0;
  if ((rc = d->d_imgs.alloc(ctx, n))) return rc;
  if (shared_tab) {
    if ((rc = ctx_put(ctx, d->d_imgs, job->imgs.data(), n * sizeof(BlendImg)))) return rc;
  } else {
    if ((rc = d->d_tab.alloc(ctx, std::max<size_t>(job->tab.size(), 1)))) return rc;
    void* dsts[2] = {d->d_imgs, d->d_tab};
    const void* srcs[2] = {job->imgs.data(), job->tab.data()};
    size_t sizes[2] = {n * sizeof(BlendImg), job->tab.size() * sizeof(double)};
    if ((rc = ctx_put_many(ctx, 2, dsts, srcs, sizes))) return rc;
  }
  const double* tab = shared_tab ? shared_tab : d->d_tab.get();
  job->g.col_sin = tab; job->g.col_cos = tab + job->ncol; job->g.row_tan = tab + 2 * job->ncol;
  if (bands == 0) return PANO_OK;
  const size_t roi = (size_t)job->roi_floats;
  if ((rc = d->d_cur.alloc(ctx, roi))) return rc;
  if ((rc = d->d_next.alloc(ctx, roi))) return rc;
  if ((rc = d->d_mask.alloc(ctx, (size_t)job->mask_bytes))) return rc;
  const size_t strip_px = (size_t)tw * (row1 - row0);
  // the weight map is needed wherever a clipped ROI has pixels on the canvas
  d->wrow0 = std::max(0, std::max(row0 - job->halo, job->clip0));
  d->wrow1 = std::min(th, job->strip ? row1 + job->halo : th);
  if ((rc = d->d_tmask.alloc(ctx, strip_px))) return rc;
  // plane table of the blur launches: (image, channel) -> offset, size; tiles of 64x32
  d->n_planes = 4 * n;
  std::vector<MbPlane> planes(d->n_planes);
  std::vector<int2> span(d->n_planes);
  for (int k = 0; k < n; ++k)
    for (int ch = 0; ch < 4; ++ch) {
      const BlendImg& im = job->imgs[k];
      planes[4 * k + ch] = MbPlane{im.roi_off + ch * im.plane, im.rw, im.rh, im.pitch, 0};
      span[4 * k + ch] = make_int2(d->n_tiles, ceil_div(im.rw, BT_W));
      d->n_tiles += ceil_div(im.rw, BT_W) * ceil_div(im.rh, BT_H);
    }
  if (bands > 1) {
    if ((rc = d->d_planes.alloc(ctx, d->n_planes))) return rc;
    if ((rc = d->d_span.alloc(ctx, d->n_planes))) return rc;
    if ((rc = ctx_put(ctx, d->d_planes, planes.data(), d->n_planes * sizeof(MbPlane)))) return rc;
    if ((rc = ctx_put(ctx, d->d_span, span.data(), d->n_planes * sizeof(int2)))) return rc;
  }
  // TMA descriptors: one per (plane, level buffer, distinct window half-width)
  for (auto& bt : job->level_taps)
    if ((bt.center == 6 || bt.center == 9) && std::find(d->centers.begin(), d->centers.end(), bt.center) == d->centers.end())
      d->centers.push_back(bt.center);
  if (!d->centers.empty()) {
    std::vector<TmaDesc> maps((size_t)d->centers.size() * 2 * d->n_planes);
    for (size_t ci = 0; ci < d->centers.size(); ++ci)
      for (int buf = 0; buf < 2; ++buf)
        for (int q = 0; q < d->n_planes; ++q) {
          const MbPlane& pl = planes[q];
          const int C = d->centers[ci];
          unsigned long long dims[2] = {(unsigned long long)pl.w, (unsigned long long)pl.h};
          unsigned long long strides[1] = {(unsigned long long)pl.pitch * sizeof(float)};
          unsigned box[2] = {(unsigned)(BT_W + 2 * ((C + 3) & ~3)), (unsigned)(BT_H + 2 * C)};
          if ((rc = ctx_tma_encode(ctx, &maps[(ci * 2 + buf) * d->n_planes + q], (buf ? d->d_next : d->d_cur) + pl.off, 2,
                                   dims, strides, box)))
            return rc;
        }
    if ((rc = d->d_maps.alloc(ctx, maps.size()))) return rc;
    if ((rc = ctx_put(ctx, d->d_maps, maps.data(), maps.size() * sizeof(TmaDesc)))) return rc;
  }
  return PANO_OK;
}

// multiband.cc:59-151 after create_first_level: the weight map, then per level blur + accumulate
// into rows [row0, row1) of d_out.  Every image's first level must be in d_cur.
static int mb_levels(pano_ctx* ctx, const BlendJob& job, BlendDev* d, int bands, float* d_out, int row0, int row1) {
  const int n = (int)job.imgs.size(), tw = job.tw;
  const dim3 b(32, 8);
  dim3 gw(ceil_div(tw, 32), ceil_div(d->wrow1 - d->wrow0, 8)), gs(ceil_div(tw, 32), ceil_div(row1 - row0, 8));
  PANO_LAUNCH(ctx, "k_mb_weight_argmax", k_mb_weight_argmax, gw, b, 0, d->d_imgs, n, d->d_cur, tw, d->wrow0, d->wrow1);
  float *cur = d->d_cur, *next = d->d_next;
  int buf = 0;     // which level buffer `cur` currently is (0: the first allocation)
  for (int level = 0; level < bands; ++level) {
    int is_last = level == bands - 1;
    if (!is_last) {
      const BlurTaps& bt = job.level_taps[level];
      const int c = bt.center;
      cudaError_t e = cudaSuccess;
      ctx->launches++;
      if (ctx->profiling) ctx_prof_begin(ctx, "k_mb_blur");
      auto ci = std::find(d->centers.begin(), d->centers.end(), c);
      if (ci != d->centers.end()) {
        const TmaDesc* maps = d->d_maps + ((size_t)(ci - d->centers.begin()) * 2 + buf) * d->n_planes;
        const int grid = std::min(d->n_tiles, ctx->num_sms * 4);
        e = c == 6 ? launch_mb_blur_tma<6>(ctx, grid, d->d_planes, d->d_span, d->n_planes, d->n_tiles, maps, next, bt)
                   : launch_mb_blur_tma<9>(ctx, grid, d->d_planes, d->d_span, d->n_planes, d->n_tiles, maps, next, bt);
      } else {
        const size_t smem = sizeof(float) * ((size_t)(MB_TH + 2 * c) * (MB_TW + 2 * c) + (size_t)MB_TH * (MB_TW + 2 * c));
        if (smem > 200 * 1024) {
          if (ctx->profiling) ctx_prof_end(ctx);
          return ctx_fail(ctx, PANO_ERR_INVALID, "blend: gaussian window %d too wide", 2 * c + 1);
        }
        e = cudaFuncSetAttribute(k_mb_blur_generic, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) {
          k_mb_blur_generic<<<d->n_tiles, 256, smem, ctx->stream>>>(d->d_planes, d->d_span, d->n_planes, cur, next, bt);
          e = cudaGetLastError();
        }
      }
      if (ctx->profiling) ctx_prof_end(ctx);
      if (e != cudaSuccess) return ctx_cuda(ctx, e, "k_mb_blur");
    }
    PANO_LAUNCH(ctx, "k_mb_accumulate", k_mb_accumulate, gs, b, 0, d->d_imgs, n, cur, next, d->d_mask, level == 0 ? 1 : 0,
              is_last, d_out, d->d_tmask, tw, row0, row1);
    if (!is_last) { std::swap(cur, next); buf ^= 1; }
  }
  return PANO_OK;
}

template <class Src>
static int blend_run(pano_ctx* ctx, const BlendJob& job, BlendDev* d, int bands, const pano_params* p, float* d_out,
                     int row0, int row1) {
  const int n = (int)job.imgs.size(), tw = job.tw;
  const dim3 b(32, 8);   // 256 threads: the 8-bit kernels' conversion table
  if (bands == 0) {
    dim3 gs(ceil_div(tw, 32), ceil_div(row1 - row0, 8));
    PANO_LAUNCH(ctx, src_name<Src>(SRC_NAMES("k_linear_blend")), k_linear_blend<Src>, gs, b, 0, d->d_imgs, n, job.g,
                p->lazy_read, p->ordered_input, d_out, tw, row0, row1);
    return PANO_OK;
  }
  dim3 gr(ceil_div(job.max_rw, 32), ceil_div(job.max_rh, 8), n);
  PANO_LAUNCH(ctx, src_name<Src>(SRC_NAMES("k_mb_first_level")), k_mb_first_level<Src>, gr, b, 0, d->d_imgs, job.g,
              d->d_cur, d->d_mask);
  return mb_levels(ctx, job, d, bands, d_out, row0, row1);
}

// pix / channels: 8-bit device sources (pano_blend_rgb8_dev, pano_blend_rows_rgb8_dev), else null and
// imgs[k].rgb_hwc are the sources
static int blend_device(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                        const pano_params* p, float* d_out, int ow, int oh, int row0, int row1,
                        const unsigned char* const* pix = nullptr, const int* channels = nullptr) {
  if (!ctx || n <= 0 || !imgs || !g || !p || !d_out || bands < 0) return PANO_ERR_INVALID;
  if (n > PANO_MAX_IMAGES)   // images on gridDim.z of k_mb_first_level
    return ctx_fail(ctx, PANO_ERR_INVALID, "blend: %d images (limit %d)", n, PANO_MAX_IMAGES);
  if (row0 < 0 || row1 > oh || row0 > row1)
    return ctx_fail(ctx, PANO_ERR_INVALID, "blend: rows [%d, %d) outside the %d-row canvas", row0, row1, oh);
  if (row0 == row1) return PANO_OK;
  BlendJob job;
  int rc = blend_plan(ctx, n, imgs, g, bands, p, ow, oh, row0, row1, !pix, &job, pix, channels);
  if (rc) return rc;
  if (job.imgs.empty()) {                              // no image reaches the strip
    size_t nfl = (size_t)job.tw * (row1 - row0) * 3;
    PANO_LAUNCH(ctx, "k_fill", k_fill, (unsigned)((nfl + 255) / 256), 256, 0, d_out, nfl, -1.f);
    return PANO_OK;
  }
  BlendDev dev;
  if ((rc = blend_dev_setup(ctx, &job, bands, row0, row1, &dev))) return rc;
  return with_reader(src_reader(pix ? channels : nullptr, n), [&](auto tag) {
    return blend_run<typename decltype(tag)::type>(ctx, job, &dev, bands, p, d_out, row0, row1);
  });
}

// ------------------------------------------------------------------ blend stream
// LAZY_READ's memory contract (blender.cc:38-64, multiband.cc:27,49): sources arrive window by
// window and are dropped after their window.  State: the canvas (linear: sums + weight plane;
// multiband: BlendDev's level buffers and masks) plus at most two windows of host sources in the
// upload ring (common.cuh): window k's upload runs while window k-1's kernels run.
// A stream of rows [row0, row1) keeps the canvas state of those rows only (blend_plan's strip
// clipping for multiband) and reads only the sources of the images that reach them.
struct pano_blend_stream {
  Sticky st;                   // every failure is sticky: the canvas state is undefined after it
  int n = 0, bands = 0, lazy = 0, ordered = 0;
  int row0 = 0, row1 = 0;
  BlendJob job;
  BlendDev dev;
  std::vector<int> slot;       // per image: its entry of job.imgs, or -1 if the rows do not need it
  DevBuf<float> d_sum;         // linear: tw×rows×3 Σ c·w
  DevBuf<float> d_wsum;        // linear: tw×rows Σ w
  // cylinder streams (pano_blend_stream_create_cyl), else empty: sources are unwarped and read through SrcCyl
  std::vector<CylImg> cyl;     // per entry of job.imgs: the warp's constants and its tables in d_cyl_tab
  DevBuf<CylImg> d_cyl;        // per entry, with its source pointer: written by the add of its window
  DevBuf<double> d_cyl_tab;    // col_x then col_cos of every image, 16 B per warped column
  int added = 0;
  UploadRing ring;
};

template <class Src>
static int stream_launch(pano_blend_stream* s, const BlendImg* d_win, const BlendImg* win, int count) {
  pano_ctx* ctx = s->st.ctx;
  const BlendJob& job = s->job;
  const dim3 b(32, 8);
  if (s->bands == 0) {
    // bounding rectangle of the window on the canvas (inclusive ranges: a superset of both range rules)
    int x0 = INT_MAX, y0 = INT_MAX, x1 = 0, y1 = 0;
    for (int k = 0; k < count; ++k) {
      x0 = std::min(x0, win[k].x0); y0 = std::min(y0, win[k].y0);
      x1 = std::max(x1, win[k].x1 + 1); y1 = std::max(y1, win[k].y1 + 1);
    }
    x1 = std::min(x1, job.tw); y0 = std::max(y0, s->row0); y1 = std::min(y1, s->row1);
    if (x0 >= x1 || y0 >= y1) return PANO_OK;
    dim3 g(ceil_div(x1 - x0, 32), ceil_div(y1 - y0, 8));
    PANO_LAUNCH(ctx, src_name<Src>(SRC_NAMES("k_linear_accumulate")), k_linear_accumulate<Src>, g, b, 0, d_win, count,
                job.g, s->lazy, s->ordered, s->d_sum, s->d_wsum, job.tw, s->row0, x0, y0, x1, y1);
  } else {
    int rw = 0, rh = 0;
    for (int k = 0; k < count; ++k) { rw = std::max(rw, win[k].rw); rh = std::max(rh, win[k].rh); }
    dim3 g(ceil_div(rw, 32), ceil_div(rh, 8), count);
    PANO_LAUNCH(ctx, src_name<Src>(SRC_NAMES("k_mb_first_level")), k_mb_first_level<Src>, g, b, 0, d_win, job.g,
                s->dev.d_cur, s->dev.d_mask);
  }
  return PANO_OK;
}

static int stream_resolve(pano_blend_stream* s, float* d_out) {
  pano_ctx* ctx = s->st.ctx;
  const size_t npx = (size_t)s->job.tw * (s->row1 - s->row0);
  if (s->bands > 0 && s->job.imgs.empty()) {          // no image reaches the rows
    PANO_LAUNCH(ctx, "k_fill", k_fill, (unsigned)((npx * 3 + 255) / 256), 256, 0, d_out, npx * 3, -1.f);
    return PANO_OK;
  }
  if (s->bands > 0) return mb_levels(ctx, s->job, &s->dev, s->bands, d_out, s->row0, s->row1);
  PANO_LAUNCH(ctx, "k_linear_resolve", k_linear_resolve, (unsigned)((npx + 255) / 256), 256, 0, s->d_sum, s->d_wsum,
              d_out, npx, s->lazy);
  return PANO_OK;
}

int blend_stream_open(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                      const pano_params* p, int ow, int oh, int row0, int row1, const double* shared_tab,
                      pano_blend_stream** out) {
  if (!ctx || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  if (n <= 0 || !imgs || !g || !p || bands < 0) return ctx_fail(ctx, PANO_ERR_INVALID, "blend stream: bad argument");
  if (n > PANO_MAX_IMAGES)   // a window's images on gridDim.z of k_mb_first_level
    return ctx_fail(ctx, PANO_ERR_INVALID, "blend stream: %d images (limit %d)", n, PANO_MAX_IMAGES);
  if (row0 < 0 || row1 > oh || row0 >= row1)
    return ctx_fail(ctx, PANO_ERR_INVALID, "blend stream: rows [%d, %d) are no strip of the %d-row canvas", row0, row1, oh);
  std::unique_ptr<pano_blend_stream> s(new pano_blend_stream);
  s->st.ctx = ctx; s->n = n; s->bands = bands; s->lazy = p->lazy_read; s->ordered = p->ordered_input;
  s->row0 = row0; s->row1 = row1;
  int rc = blend_plan(ctx, n, imgs, g, bands, p, ow, oh, row0, row1, false, &s->job, nullptr, nullptr, !shared_tab);
  if (!rc && !s->job.imgs.empty()) rc = blend_dev_setup(ctx, &s->job, bands, row0, row1, &s->dev, shared_tab);
  if (rc) return rc;
  s->slot.assign(n, -1);
  for (size_t q = 0; q < s->job.imgs.size(); ++q) {
    const int k = s->job.src[q];
    if (blend_strip_reads(imgs[k], bands, s->job.halo, oh, row0, row1)) s->slot[k] = (int)q;
  }
  if (bands == 0) {
    const size_t npx = (size_t)ow * (row1 - row0);
    if ((rc = s->d_sum.alloc(ctx, npx * 3)) || (rc = s->d_wsum.alloc(ctx, npx))) return rc;
    PANO_LAUNCH(ctx, "k_fill", k_fill, (unsigned)((npx * 3 + 255) / 256), 256, 0, s->d_sum, npx * 3, 0.f);
    PANO_LAUNCH(ctx, "k_fill", k_fill, (unsigned)((npx + 255) / 256), 256, 0, s->d_wsum, npx, 0.f);
  }
  *out = s.release();
  return PANO_OK;
}

int blend_sweep_tables(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                       const pano_params* p, int ow, int oh, std::vector<double>* tab) {
  BlendJob job;
  if (int rc = blend_plan(ctx, n, imgs, g, bands, p, ow, oh, 0, oh, false, &job)) return rc;
  tab->swap(job.tab);
  return PANO_OK;
}

int cyl_tabs(pano_ctx* ctx, int n, const pano_blend_image* imgs, const int* src_w, const int* src_h, double h_factor,
             const pano_params* p, CylTabs* ct) {
  if (n <= 0 || !imgs || !src_w || !src_h || !p)
    return ctx_fail(ctx, PANO_ERR_INVALID, "cylinder blend stream: bad argument");
  if (n > PANO_MAX_IMAGES)
    return ctx_fail(ctx, PANO_ERR_INVALID, "blend stream: %d images (limit %d)", n, PANO_MAX_IMAGES);
  // the warp of every source (host arithmetic, as pano_cyl_warp_batch_dev does it) must be the image blended
  ct->maps.resize(n);
  ct->off.resize(n);
  ct->w.assign(src_w, src_w + n);
  ct->h.assign(src_h, src_h + n);
  ct->tabs.clear();
  for (int k = 0; k < n; ++k) {
    if (src_w[k] < 2 || src_h[k] < 2)
      return ctx_fail(ctx, PANO_ERR_INVALID, "cylinder blend stream: source %d is %dx%d, under 2x2", k, src_w[k],
                      src_h[k]);
    ct->off[k] = ct->tabs.size();
    if (!cyl_map(src_w[k], src_h[k], h_factor, p, nullptr, 0, &ct->maps[k], &ct->tabs))
      return ctx_fail(ctx, PANO_ERR_INVALID, "cylinder radius <= 0");
    if (ct->maps[k].ow != imgs[k].w || ct->maps[k].oh != imgs[k].h)
      return ctx_fail(ctx, PANO_ERR_INVALID,
                      "cylinder blend stream: image %d is %dx%d but its %dx%d source warps to %dx%d", k, imgs[k].w,
                      imgs[k].h, src_w[k], src_h[k], ct->maps[k].ow, ct->maps[k].oh);
  }
  return PANO_OK;
}

int blend_stream_open_cyl(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                          const pano_params* p, int ow, int oh, int row0, int row1, const double* shared_tab,
                          const CylTabs& ct, const double* d_cyl_tab, pano_blend_stream** out) {
  pano_blend_stream* raw = nullptr;
  if (int rc = blend_stream_open(ctx, n, imgs, g, bands, p, ow, oh, row0, row1, shared_tab, &raw)) return rc;
  std::unique_ptr<pano_blend_stream> s(raw);
  const size_t ne = s->job.imgs.size();
  int rc = 0;
  if (!d_cyl_tab) {
    if ((rc = s->d_cyl_tab.alloc(ctx, std::max<size_t>(ct.tabs.size(), 1)))) return rc;
    if ((rc = ctx_put(ctx, s->d_cyl_tab, ct.tabs.data(), ct.tabs.size() * sizeof(double)))) return rc;
    d_cyl_tab = s->d_cyl_tab;
  }
  if ((rc = s->d_cyl.alloc(ctx, std::max<size_t>(ne, 1)))) return rc;
  s->cyl.resize(ne);
  for (size_t q = 0; q < ne; ++q) {
    const int k = s->job.src[q];
    const CylMap& m = ct.maps[k];
    CylImg& c = s->cyl[q];
    memset(&c, 0, sizeof(c));
    c.w = ct.w[k]; c.h = ct.h[k];
    c.col_x = d_cyl_tab + ct.off[k];
    c.col_cos = c.col_x + m.ow;
    c.r = m.r; c.cy = m.cy; c.offy = m.offy; c.sizefactor_inv = m.sizefactor_inv;
  }
  *out = s.release();
  return PANO_OK;
}

extern "C" {

int pano_blend_target_size(int n, const pano_blend_image* imgs, int* ow, int* oh) {
  if (n <= 0 || !imgs || !ow || !oh) return PANO_ERR_INVALID;
  int tw = 0, th = 0;
  for (int k = 0; k < n; ++k) { tw = std::max(tw, imgs[k].x1); th = std::max(th, imgs[k].y1); }
  *ow = tw; *oh = th;
  return PANO_OK;
}

int pano_blend_dev(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                   const pano_params* p, float* d_out, int ow, int oh) {
  ctx_enter(ctx);
  return blend_device(ctx, n, imgs, g, bands, p, d_out, ow, oh, 0, oh);
}

int pano_blend_rgb8_dev(pano_ctx* ctx, int n, const pano_blend_image* imgs, const unsigned char* const* d_pix,
                        const int* channels, const pano_blend_geom* g, int bands, const pano_params* p, float* d_out,
                        int ow, int oh) {
  ctx_enter(ctx);
  if (!ctx) return PANO_ERR_INVALID;
  if (!d_pix || !channels) return ctx_fail(ctx, PANO_ERR_INVALID, "blend rgb8: null source list");
  return blend_device(ctx, n, imgs, g, bands, p, d_out, ow, oh, 0, oh, d_pix, channels);
}

int pano_blend_rows_dev(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                        const pano_params* p, float* d_out_rows, int ow, int oh, int row0, int row1) {
  ctx_enter(ctx);
  return blend_device(ctx, n, imgs, g, bands, p, d_out_rows, ow, oh, row0, row1);
}

int pano_blend_rows_rgb8_dev(pano_ctx* ctx, int n, const pano_blend_image* imgs, const unsigned char* const* d_pix,
                             const int* channels, const pano_blend_geom* g, int bands, const pano_params* p,
                             float* d_out_rows, int ow, int oh, int row0, int row1) {
  ctx_enter(ctx);
  if (!ctx) return PANO_ERR_INVALID;
  if (!d_pix || !channels) return ctx_fail(ctx, PANO_ERR_INVALID, "blend rows rgb8: null source list");
  return blend_device(ctx, n, imgs, g, bands, p, d_out_rows, ow, oh, row0, row1, d_pix, channels);
}

int pano_blend_stream_create(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                             const pano_params* p, int ow, int oh, pano_blend_stream** out) {
  ctx_enter(ctx);
  return blend_stream_open(ctx, n, imgs, g, bands, p, ow, oh, 0, oh, nullptr, out);
}

int pano_blend_stream_create_rows(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g,
                                  int bands, const pano_params* p, int ow, int oh, int row0, int row1,
                                  pano_blend_stream** out) {
  ctx_enter(ctx);
  return blend_stream_open(ctx, n, imgs, g, bands, p, ow, oh, row0, row1, nullptr, out);
}

int pano_blend_stream_create_cyl(pano_ctx* ctx, int n, const pano_blend_image* imgs, const int* src_w,
                                 const int* src_h, double h_factor, const pano_blend_geom* g, int bands,
                                 const pano_params* p, int ow, int oh, pano_blend_stream** out) {
  ctx_enter(ctx);
  if (!ctx || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  CylTabs ct;
  if (int rc = cyl_tabs(ctx, n, imgs, src_w, src_h, h_factor, p, &ct)) return rc;
  return blend_stream_open_cyl(ctx, n, imgs, g, bands, p, ow, oh, 0, oh, nullptr, ct, nullptr, out);
}

int pano_blend_stream_needs(const pano_blend_stream* s, unsigned char* flags) {
  if (!s) return PANO_ERR_INVALID;
  ctx_enter(s->st.ctx);
  if (!flags) return ctx_fail(s->st.ctx, PANO_ERR_INVALID, "blend stream: null flags");
  for (int k = 0; k < s->n; ++k) flags[k] = s->slot[k] >= 0 ? 1 : 0;
  return PANO_OK;
}

int pano_blend_stream_add(pano_blend_stream* s, int first, int count, const void* const* srcs, int kind, int channels) {
  if (!s) return PANO_ERR_INVALID;
  pano_ctx* ctx = s->st.ctx;
  ctx_enter(ctx);
  SrcKind sk;
  if (int rc = s->st.add_check("blend stream", s->n, s->added, first, count, s->n, srcs, s->slot.data(), kind,
                               channels, &sk))
    return rc;
  // The window's needed images.  Their table rows go to d_imgs from the first one's entry on: for multiband
  // they are exactly the consecutive entries mb_levels reads again; linear reads them in this window only.
  // A cylinder stream's entries point at their warp entries in d_cyl, and those at the sources.
  const bool cyl = !s->cyl.empty();
  std::vector<BlendImg> win;
  std::vector<CylImg> cwin;
  std::vector<const void*> wsrc;
  std::vector<size_t> bytes;
  int j0 = -1;
  for (int k = 0; k < count; ++k) {
    const int q = s->slot[first + k];
    if (q < 0) continue;
    if (j0 < 0) j0 = q;
    win.push_back(s->job.imgs[q]);
    win.back().channels = channels;
    if (cyl) {
      cwin.push_back(s->cyl[q]);
      cwin.back().channels = channels;
      win.back().src = s->d_cyl + q;
      bytes.push_back(src_bytes(cwin.back().w, cwin.back().h, sk.u8, channels));
    } else {
      bytes.push_back(src_bytes(win.back().w, win.back().h, sk.u8, channels));
    }
    wsrc.push_back(srcs[k]);
  }
  const int nw = (int)win.size();
  if (nw == 0) {
    s->added += count;
    return PANO_OK;
  }
  int slot = -1, rc = 0;
  std::vector<const void*> d_src(wsrc);   // host sources: their copies in the ring
  if (sk.host && (rc = s->ring.upload(ctx, "blend stream", nw, wsrc.data(), bytes.data(), d_src.data(), &slot)))
    return s->st.fail(rc);
  for (int k = 0; k < nw; ++k) (cyl ? cwin[k].src : win[k].src) = d_src[k];
  BlendImg* d_win = s->dev.d_imgs + j0;
  if (cyl) {
    void* dsts[2] = {d_win, s->d_cyl + j0};
    const void* hsrcs[2] = {win.data(), cwin.data()};
    size_t sizes[2] = {nw * sizeof(BlendImg), nw * sizeof(CylImg)};
    if ((rc = ctx_put_many(ctx, 2, dsts, hsrcs, sizes))) return s->st.fail(rc);
  } else {
    if ((rc = ctx_put(ctx, d_win, win.data(), nw * sizeof(BlendImg)))) return s->st.fail(rc);
  }
  rc = with_reader(src_reader(sk.u8 ? &channels : nullptr, 1), [&](auto tag) {
    using Src = typename decltype(tag)::type;
    return cyl ? stream_launch<SrcCyl<Src>>(s, d_win, win.data(), nw) : stream_launch<Src>(s, d_win, win.data(), nw);
  });
  if (rc) return s->st.fail(rc);
  if (slot >= 0 && (rc = s->st.cuda(s->ring.release(ctx, slot), "s->ring.release(ctx, slot)"))) return rc;
  s->added += count;
  return PANO_OK;
}

int pano_blend_stream_finish_dev(pano_blend_stream* s, float* d_out) {
  if (!s) return PANO_ERR_INVALID;
  ctx_enter(s->st.ctx);
  if (int rc = s->st.finish_check("blend stream", d_out, s->added, s->n)) return rc;
  if (int rc = stream_resolve(s, d_out)) return s->st.fail(rc);
  return PANO_OK;
}

int pano_blend_stream_finish(pano_blend_stream* s, float* out) {
  if (!s) return PANO_ERR_INVALID;
  pano_ctx* ctx = s->st.ctx;
  ctx_enter(ctx);
  int rc = s->st.finish_check("blend stream", out, s->added, s->n);
  if (rc) return rc;
  const size_t nfl = (size_t)s->job.tw * (s->row1 - s->row0) * 3;
  DevBuf<float> d_tmp;
  float* d_out = s->d_sum;     // linear: resolved in place
  if (s->bands > 0) {
    if ((rc = d_tmp.alloc(ctx, nfl))) return s->st.fail(rc);
    d_out = d_tmp;
  }
  if ((rc = stream_resolve(s, d_out))) return s->st.fail(rc);
  if ((rc = s->st.cuda(cudaMemcpyAsync(out, d_out, nfl * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream),
                       "cudaMemcpyAsync(out, d_out, nfl * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream)")) ||
      (rc = s->st.cuda(cudaStreamSynchronize(ctx->stream), "cudaStreamSynchronize(ctx->stream)")))
    return rc;
  d_tmp.reset();
  return PANO_OK;
}

void pano_blend_stream_free(pano_blend_stream* s) {
  if (s) ctx_enter(s->st.ctx);
  delete s;
}

int pano_blend(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
               const pano_params* p, float* out, int ow, int oh) {
  ctx_enter(ctx);
  if (!ctx || n <= 0 || !imgs || !out) return PANO_ERR_INVALID;
  if (n > PANO_MAX_IMAGES) return ctx_fail(ctx, PANO_ERR_INVALID, "blend: %d images (limit %d)", n, PANO_MAX_IMAGES);
  std::vector<pano_blend_image> dimgs(imgs, imgs + n);
  std::vector<DevBuf<float>> bufs(n);
  int rc = 0;
  for (int k = 0; k < n; ++k) {
    if (!imgs[k].rgb_hwc || imgs[k].w <= 0 || imgs[k].h <= 0) return ctx_fail(ctx, PANO_ERR_INVALID, "blend: image %d empty", k);
    const size_t nfl = (size_t)imgs[k].w * imgs[k].h * 3;
    if ((rc = bufs[k].alloc(ctx, nfl))) return rc;
    PANO_CUDA(ctx, cudaMemcpyAsync(bufs[k], imgs[k].rgb_hwc, nfl * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    dimgs[k].rgb_hwc = bufs[k];
  }
  const size_t nfl = (size_t)std::max(ow, 0) * std::max(oh, 0) * 3;
  DevBuf<float> d_out;
  if ((rc = d_out.alloc(ctx, nfl))) return rc;
  if ((rc = blend_device(ctx, n, dimgs.data(), g, bands, p, d_out, ow, oh, 0, oh))) return rc;
  PANO_CUDA(ctx, cudaMemcpyAsync(out, d_out, nfl * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PANO_OK;
}

}  // extern "C"
