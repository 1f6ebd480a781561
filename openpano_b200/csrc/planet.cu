// planet.cu — the "little planet" (stereographic) view of a mosaic.
//
// Replaces planet() (main.cc:294-331, the `planet` sub-command at :352-353) without its file I/O:
// a PANO_PLANET_SIZE² (1000×1000) image whose pixel (i, j) samples the mosaic at
//   row    = min(h - (hypot(center - i, center - j) / center) * h, h - 1)
//   column = theta(i, j) / (2π) * w
// with one bilinear interpolate (lib/imgproc.cc:135-156).  hypot and atan are the only libm calls,
// and both depend on (i, j) alone: the host evaluates them once per process with the libm the
// reference calls and stores d / center and theta / (2π) per pixel (the rule DESIGN.md §3 applies
// to the warp's tan/cos tables).  Each context uploads that table on its first planet call and keeps
// it until pano_destroy; the kernel then does only IEEE double arithmetic and the f32 gather.
// pano_planet_pix8[_dev] take the decoded 8-bit image instead (any PANO_PIX_* format) and convert each tap as
// read_img converts it, so `planet` runs from the file's pixels without an f32 copy of the mosaic.
#include "common.cuh"
#include <math.h>
#include <vector>

namespace {

constexpr int kSize = PANO_PLANET_SIZE, kCenter = PANO_PLANET_SIZE / 2;   // main.cc:297 OUTSIZE, center
constexpr size_t kPixels = (size_t)kSize * kSize;

// x = d / center (main.cc:302-304), y = theta / (M_PI * 2) (:308-323, left operand of `* w`);
// x = -1 marks the pixels the loop skips (d >= center || d == 0).
const std::vector<double2>& planet_table() {
  static const std::vector<double2> tab = [] {
    std::vector<double2> t(kPixels);
    for (int i = 0; i < kSize; ++i)
      for (int j = 0; j < kSize; ++j) {
        double2& e = t[(size_t)i * kSize + j];
        const double d = hypot((double)(kCenter - i), (double)(kCenter - j));
        if (d >= kCenter || d == 0) { e.x = -1.0; e.y = 0.0; continue; }
        double theta;
        if (j == kCenter) {
          theta = i < kCenter ? M_PI / 2 : 3 * M_PI / 2;
        } else {
          theta = atan((double)(kCenter - i) / (kCenter - j));
          if (theta < 0) theta += M_PI;
          if ((theta == 0) && (j > kCenter)) theta += M_PI;
          if (kCenter < i) theta += M_PI;
        }
        e.x = d / kCenter;
        e.y = theta / (M_PI * 2);
      }
    return t;
  }();
  return tab;
}

int planet_table_dev(pano_ctx* ctx, const double2** out) {
  if (!ctx->planet_tab) {
    DevBuf<double2> tab;
    if (int rc = tab.alloc(ctx, kPixels)) return rc;
    cudaError_t e = cudaMemcpyAsync(tab, planet_table().data(), kPixels * sizeof(double2), cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) return ctx_cuda(ctx, e, "planet table upload");
    ctx->planet_tab = std::move(tab);
  }
  *out = ctx->planet_tab;
  return PANO_OK;
}

}  // namespace

// one thread per output pixel (main.cc:301-329); every pixel is written, -1 where nothing maps.  Src is the
// tap reader (common.cuh): every tap it returns is the f32 value read_img's image holds, so the planet of 8-bit
// pixels is the planet of that image, bit for bit.
template <class Src>
__device__ __forceinline__ void planet_px(const double2* __restrict__ tab, const Src& src, int w, int h,
                                          float* __restrict__ dst) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= kSize || i >= kSize) return;
  const size_t k = (size_t)i * kSize + j;
  const double2 t = __ldg(tab + k);
  float o0 = -1.f, o1 = -1.f, o2 = -1.f;
  if (t.x >= 0) {
    const double hd = (double)h;
    double dist = hd - t.x * hd;                 // :306
    const double theta = t.y * (double)w;        // :323
    if (hd - 1 < dist) dist = hd - 1;            // :325 update_min
    float c0, c1, c2;
    if (interpolate_rgb(src, w, h, (float)dist, (float)theta, &c0, &c1, &c2)) { o0 = c0; o1 = c1; o2 = c2; }
  }
  float* p = dst + k * 3;
  p[0] = o0; p[1] = o1; p[2] = o2;
}

// an h×w×3 f32 image
__global__ void k_planet(const double2* __restrict__ tab, const float* __restrict__ src, int w, int h,
                         float* __restrict__ dst) {
  planet_px(tab, SrcF32{src}, w, h, dst);
}

// 8-bit pixels in format fmt (PANO_PIX_*): Src = SrcRgb8 for grey and interleaved RGB, SrcPix8 for RGBA and planar
template <class Src>
__global__ void k_planet8(const double2* __restrict__ tab, const unsigned char* __restrict__ pix, int fmt, int w, int h,
                          float* __restrict__ dst) {
  __shared__ float lut[256];
  build_rgb8_lut(lut, threadIdx.y * blockDim.x + threadIdx.x);   // all 256 threads, before any leaves at the edge
  __syncthreads();
  planet_px(tab, Src::at(pix, w, h, fmt, lut), w, h, dst);
}

extern "C" {

int pano_planet_dev(pano_ctx* ctx, const float* d_rgb_hwc, int w, int h, float* d_out_hwc) {
  ctx_enter(ctx);
  if (!ctx) return PANO_ERR_INVALID;
  if (!d_rgb_hwc || !d_out_hwc || w < 1 || h < 1)
    return ctx_fail(ctx, PANO_ERR_INVALID, "planet: null pointer or empty %dx%d input", w, h);
  const double2* tab = nullptr;
  int rc = planet_table_dev(ctx, &tab);
  if (rc) return rc;
  dim3 b(32, 8), g(ceil_div(kSize, 32), ceil_div(kSize, 8));
  PANO_LAUNCH(ctx, "k_planet", k_planet, g, b, 0, tab, d_rgb_hwc, w, h, d_out_hwc);
  return PANO_OK;
}

int pano_planet(pano_ctx* ctx, const float* rgb_hwc, int w, int h, float* out_hwc) {
  ctx_enter(ctx);
  if (!ctx) return PANO_ERR_INVALID;
  if (!rgb_hwc || !out_hwc || w < 1 || h < 1)
    return ctx_fail(ctx, PANO_ERR_INVALID, "planet: null pointer or empty %dx%d input", w, h);
  const size_t ns = (size_t)w * h * 3, nd = (size_t)kPixels * 3;
  DevBuf<float> d_src, d_dst;
  int rc = 0;
  if ((rc = d_src.alloc(ctx, ns)) || (rc = d_dst.alloc(ctx, nd))) return rc;
  PANO_CUDA(ctx, cudaMemcpyAsync(d_src, rgb_hwc, ns * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = pano_planet_dev(ctx, d_src, w, h, d_dst))) return rc;
  PANO_CUDA(ctx, cudaMemcpyAsync(out_hwc, d_dst, nd * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PANO_OK;
}

int pano_planet_pix8_dev(pano_ctx* ctx, const unsigned char* d_pix, int format, int w, int h, float* d_out_hwc) {
  ctx_enter(ctx);
  if (!ctx) return PANO_ERR_INVALID;
  if (!d_pix || !d_out_hwc || w < 1 || h < 1)
    return ctx_fail(ctx, PANO_ERR_INVALID, "planet pix8: null pointer or empty %dx%d input", w, h);
  if (int rc = pix8_check(ctx, "planet pix8", 0, format, d_pix)) return rc;
  const double2* tab = nullptr;
  int rc = planet_table_dev(ctx, &tab);
  if (rc) return rc;
  dim3 b(32, 8), g(ceil_div(kSize, 32), ceil_div(kSize, 8));   // 256 threads: the 8-bit conversion table
  return with_reader(src_reader(&format, 1), [&](auto tag) -> int {
    using Src = typename decltype(tag)::type;
    if constexpr (Src::kLut)   // SrcF32 (f32 sources only) has no k_planet8
      PANO_LAUNCH(ctx, src_name<Src>(SRC_NAMES("k_planet")), k_planet8<Src>, g, b, 0, tab, d_pix, format, w, h, d_out_hwc);
    return PANO_OK;
  });
}

int pano_planet_pix8(pano_ctx* ctx, const unsigned char* pix, int format, int w, int h, float* out_hwc) {
  ctx_enter(ctx);
  if (!ctx) return PANO_ERR_INVALID;
  if (!pix || !out_hwc || w < 1 || h < 1)
    return ctx_fail(ctx, PANO_ERR_INVALID, "planet pix8: null pointer or empty %dx%d input", w, h);
  if (int rc = pix8_check(ctx, "planet pix8", 0, format, nullptr)) return rc;
  const size_t ns = (size_t)w * h * pix8_bytes(format), nd = (size_t)kPixels * 3;
  DevBuf<unsigned char> d_src;
  DevBuf<float> d_dst;
  int rc = 0;
  if ((rc = d_src.alloc(ctx, ns)) || (rc = d_dst.alloc(ctx, nd))) return rc;
  PANO_CUDA(ctx, cudaMemcpyAsync(d_src, pix, ns, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = pano_planet_pix8_dev(ctx, d_src, format, w, h, d_dst))) return rc;
  PANO_CUDA(ctx, cudaMemcpyAsync(out_hwc, d_dst, nd * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PANO_OK;
}

}  // extern "C"
