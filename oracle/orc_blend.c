/*
 * orc_blend.c — plain-C restatement of the reference's two blenders.
 * TEST INFRASTRUCTURE ONLY (see orc_common.h).  Citations relative to
 * the reference's src/.
 */
#include "orc_common.h"

/* The inverse map the reference hands to every blender as a std::function:
 * stitch/stitcher_image.cc:142-151 with stitch/projection.hh:14-71. */
static void coor_func(const pano_blend_image* im, const pano_blend_geom* g, int tx, int ty,
                      double* ox, double* oy) {
  double cx = tx * g->res_x + g->proj_min_x;
  double cy = ty * g->res_y + g->proj_min_y;
  double hx, hy, hz, rx, ry, rz, denom;
  const double* d = im->homo_inv;
  if (g->projection == PANO_PROJ_FLAT) { hx = cx; hy = cy; hz = 1; }
  else if (g->projection == PANO_PROJ_CYLINDRICAL) { hx = sin(cx); hy = cy; hz = cos(cx); }
  else { hx = sin(cx); hy = tan(cy); hz = cos(cx); }
  rx = d[0] * hx + d[1] * hy + d[2] * hz;
  ry = d[3] * hx + d[4] * hy + d[5] * hz;
  rz = d[6] * hx + d[7] * hy + d[8] * hz;
  if (rz < 0) { *ox = -10; *oy = -10; return; }
  denom = 1.0 / rz;
  *ox = rx * denom + im->w * 0.5;
  *oy = ry * denom + im->h * 0.5;
}

static int range_contain(const pano_blend_image* im, int r, int c) { /* blender.hh:21-24 */
  return r >= im->y0 && r <= im->y1 && c >= im->x0 && c <= im->x1;
}

/* blender.cc:27-36 GET_COLOR_AND_W; returns 0 for `continue` */
static int color_and_w(const pano_blend_image* im, const pano_blend_geom* g, int i, int j,
                       int ordered_input, float color[3], float* wout) {
  double x, y;
  float r, c, w;
  coor_func(im, g, j, i, &x, &y);
  if (x < 0 || x >= im->w || y < 0 || y >= im->h) return 0; /* blender.hh:39-44 map_coor -> NaN */
  r = (float)y; c = (float)x;
  if (!orc_interpolate(im->rgb_hwc, im->w, im->h, r, c, color)) return 0;
  if (color[0] < 0) return 0;
  w = (float)(0.5 - fabs(c / im->w - 0.5));
  if (!ordered_input) w = (float)(w * (0.5 - fabs(r / im->h - 0.5)));
  color[0] *= w; color[1] *= w; color[2] *= w;
  *wout = w;
  return 1;
}

/* stitch/blender.cc:24-96 LinearBlender::run */
static int linear_blend(int n, const pano_blend_image* imgs, const pano_blend_geom* g,
                        const pano_params* P, float* out, int tw, int th) {
  int i, j, k;
  if (P->lazy_read) {
    float* weight = (float*)calloc((size_t)tw * th, sizeof(float));
    memset(out, 0, sizeof(float) * (size_t)tw * th * 3);
    for (k = 0; k < n; ++k) {
      const pano_blend_image* im = &imgs[k];
      ORC_PAR_FOR(private(j))
      for (i = im->y0; i < im->y1; ++i)
        for (j = im->x0; j < im->x1; ++j) {
          float color[3], w;
          if (!color_and_w(im, g, i, j, P->ordered_input, color, &w)) continue;
          out[((size_t)i * tw + j) * 3] += color[0];
          out[((size_t)i * tw + j) * 3 + 1] += color[1];
          out[((size_t)i * tw + j) * 3 + 2] += color[2];
          weight[(size_t)i * tw + j] += w;
        }
    }
    ORC_PAR_FOR(private(j))
    for (i = 0; i < th; ++i)
      for (j = 0; j < tw; ++j) {
        float* p = out + ((size_t)i * tw + j) * 3;
        float w = weight[(size_t)i * tw + j];
        if (w) { p[0] /= w; p[1] /= w; p[2] /= w; }
        else { p[0] = p[1] = p[2] = -1; }
      }
    free(weight);
  } else {
    ORC_PAR_FOR(private(j, k))
    for (i = 0; i < th; ++i)
      for (j = 0; j < tw; ++j) {
        float isum[3] = {0, 0, 0}, wsum = 0;
        float* p = out + ((size_t)i * tw + j) * 3;
        p[0] = p[1] = p[2] = -1;
        for (k = 0; k < n; ++k)
          if (range_contain(&imgs[k], i, j)) {
            float color[3], w;
            if (!color_and_w(&imgs[k], g, i, j, P->ordered_input, color, &w)) continue;
            isum[0] += color[0]; isum[1] += color[1]; isum[2] += color[2];
            wsum += w;
          }
        if (wsum > 0) { /* Vector::operator/(T p) = *this * (1.0 / p), geometry.hh:117-118 */
          float inv = (float)(1.0 / wsum);
          p[0] = isum[0] * inv; p[1] = isum[1] * inv; p[2] = isum[2] * inv;
        }
      }
  }
  return 0;
}

typedef struct {
  int rw, rh;           /* ROI size = range.width(), range.height() */
  float* cur;           /* rw*rh*4: (r, g, b, w) = WeightedPixel, multiband.hh:13-23 */
  float* next;
  unsigned char* mask;  /* 1: invalid (Mask2D) */
} mb_image;

/* stitch/multiband.cc:59-151 MultiBandBlender::run (+ create_first_level :19-57,
 * update_weight_map :125-143, create_next_level :145-151).  Image order is the
 * input order (the single-thread order of the omp critical at :50-54). */
static int multiband_blend(int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                           const pano_params* P, float* out, int tw, int th) {
  mb_image* M = (mb_image*)calloc((size_t)n, sizeof(mb_image));
  unsigned char* tmask = (unsigned char*)calloc((size_t)tw * th, 1);
  int i, j, k, level;
  (void)P;
  for (k = 0; k < n; ++k) { /* create_first_level */
    const pano_blend_image* im = &imgs[k];
    mb_image* m = &M[k];
    m->rw = im->x1 - im->x0 + 1; m->rh = im->y1 - im->y0 + 1;
    m->cur = (float*)malloc(sizeof(float) * 4 * (size_t)m->rw * m->rh);
    m->next = NULL;
    m->mask = (unsigned char*)calloc((size_t)m->rw * m->rh, 1);
    ORC_PAR_FOR(private(j))
    for (i = 0; i < m->rh; ++i)
      for (j = 0; j < m->rw; ++j) {
        double x, y;
        float c[3];
        float* px = m->cur + ((size_t)i * m->rw + j) * 4;
        int ok;
        coor_func(im, g, j + im->x0, i + im->y0, &x, &y);
        ok = orc_interpolate(im->rgb_hwc, im->w, im->h, (float)y, (float)x, c);
        if (ok) { float mn = c[0] < c[1] ? c[0] : c[1]; if (c[2] < mn) mn = c[2]; if (mn < 0) ok = 0; }
        if (!ok) {
          px[0] = px[1] = px[2] = 0; px[3] = 0;
          m->mask[(size_t)i * m->rw + j] = 1;
        } else {
          double ox = x / im->w - 0.5, oy = y / im->h - 0.5, ww;
          px[0] = c[0]; px[1] = c[1]; px[2] = c[2];
          ww = (0.5f - fabs(ox)) * (0.5f - fabs(oy));
          if (ww < 0.0) ww = 0.0; /* std::max(0.0, .) */
          px[3] = (float)(ww + ORC_EPS);
        }
      }
  }
  ORC_PAR_FOR(private(j, k))
  for (i = 0; i < th; ++i) /* update_weight_map */
    for (j = 0; j < tw; ++j) {
      float mx = 0.f;
      float* maxp = NULL;
      for (k = 0; k < n; ++k)
        if (range_contain(&imgs[k], i, j)) {
          float* w = M[k].cur + ((size_t)(i - imgs[k].y0) * M[k].rw + (j - imgs[k].x0)) * 4 + 3;
          if (*w > mx) { mx = *w; maxp = w; }
          *w = 0;
        }
      if (maxp) *maxp = 1;
    }
  for (i = 0; i < th; ++i) for (j = 0; j < tw; ++j) { float* p = out + ((size_t)i * tw + j) * 3; p[0] = p[1] = p[2] = -1; }
  for (level = 0; level < bands; ++level) {
    int is_last = level == bands - 1;
    if (!is_last) { /* create_next_level */
      float sigma = (float)(sqrt(level * 2 + 1.0) * 4);
      float kernel[256];
      int kw = orc_gauss_kernel(sigma, P->gauss_window_factor, kernel);
      ORC_PAR_FOR(schedule(dynamic, 1))   /* images are independent (multiband.cc:145-151) */
      for (k = 0; k < n; ++k) {
        if (!M[k].next) M[k].next = (float*)malloc(sizeof(float) * 4 * (size_t)M[k].rw * M[k].rh);
        orc_blur(M[k].cur, M[k].next, M[k].rw, M[k].rh, 4, kernel, kw);
      }
    }
    ORC_PAR_FOR(private(j, k))
    for (i = 0; i < th; ++i)
      for (j = 0; j < tw; ++j) {
        float isum[3] = {0, 0, 0}, wsum = 0;
        float* p = out + ((size_t)i * tw + j) * 3;
        for (k = 0; k < n; ++k) {
          size_t idx;
          const float *cc, *cn;
          float w;
          if (!range_contain(&imgs[k], i, j)) continue;
          idx = (size_t)(i - imgs[k].y0) * M[k].rw + (j - imgs[k].x0);
          if (M[k].mask[idx]) continue;
          cc = M[k].cur + idx * 4;
          w = cc[3];
          if (w <= 0) continue;
          if (!is_last) {
            cn = M[k].next + idx * 4;
            isum[0] += (cc[0] - cn[0]) * w; isum[1] += (cc[1] - cn[1]) * w; isum[2] += (cc[2] - cn[2]) * w;
          } else {
            isum[0] += cc[0] * w; isum[1] += cc[1] * w; isum[2] += cc[2] * w;
          }
          wsum += w;
        }
        if (wsum < ORC_EPS) continue;
        isum[0] /= wsum; isum[1] /= wsum; isum[2] /= wsum;
        if (!tmask[(size_t)i * tw + j]) {
          p[0] = isum[0]; p[1] = isum[1]; p[2] = isum[2];
          tmask[(size_t)i * tw + j] = 1;
        } else { p[0] += isum[0]; p[1] += isum[1]; p[2] += isum[2]; }
      }
    if (!is_last) for (k = 0; k < n; ++k) { float* t = M[k].cur; M[k].cur = M[k].next; M[k].next = t; }
  }
  for (i = 0; i < th; ++i)
    for (j = 0; j < tw; ++j)
      if (tmask[(size_t)i * tw + j]) {
        float* p = out + ((size_t)i * tw + j) * 3;
        int c;
        for (c = 0; c < 3; ++c) { float v = p[c] < 1.0f ? p[c] : 1.0f; p[c] = v > 0.f ? v : 0.f; }
      }
  for (k = 0; k < n; ++k) { free(M[k].cur); free(M[k].next); free(M[k].mask); }
  free(M); free(tmask);
  return 0;
}

int orc_blend(int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
              const pano_params* P, float* out, int ow, int oh) {
  int k, tw = 0, th = 0;
  for (k = 0; k < n; ++k) { if (imgs[k].x1 > tw) tw = imgs[k].x1; if (imgs[k].y1 > th) th = imgs[k].y1; }
  if (tw != ow || th != oh) return -1;
  if (bands > 0) return multiband_blend(n, imgs, g, bands, P, out, tw, th);
  return linear_blend(n, imgs, g, P, out, tw, th);
}

#include <time.h> /* clock_gettime: built with -std=gnu11 */
static double now_s(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec + ts.tv_nsec * 1e-9; }

/* One pass of the hot path with the restated stages, single thread (see
 * oracle_api.h).  use_flann is ignored: the port only has the exact matcher. */
int orc_hotpath(int n, const float* const* rgb, const int* w, const int* h, int n_pairs, const int* ij,
                int use_flann, const pano_blend_image* bimgs, const pano_blend_geom* g, int bands,
                const pano_params* P, float* out, int ow, int oh, int* n_feat, int* n_match, double* seconds) {
  float** desc = (float**)calloc((size_t)n, sizeof(float*));
  double t = now_s();
  int k, rc = 0;
  const int cap = 65536;
  (void)use_flann;
  for (k = 0; k < n; ++k) {
    desc[k] = (float*)malloc(sizeof(float) * 128 * (size_t)cap);
    n_feat[k] = orc_sift_detect(rgb[k], w[k], h[k], P, cap, NULL, desc[k]);
    if (n_feat[k] <= 0) rc = -5;
  }
  seconds[0] = now_s() - t; t = now_s();
  for (k = 0; k < n_pairs && !rc; ++k) {
    int a = ij[2 * k], b = ij[2 * k + 1];
    int mn = n_feat[a] < n_feat[b] ? n_feat[a] : n_feat[b];
    int* pairs = (int*)malloc(sizeof(int) * 2 * (size_t)(mn + 1));
    orc_match(desc[a], n_feat[a], desc[b], n_feat[b], P, pairs, &n_match[k]);
    free(pairs);
  }
  seconds[1] = now_s() - t; t = now_s();
  if (!rc) rc = orc_blend(n, bimgs, g, bands, P, out, ow, oh);
  seconds[2] = now_s() - t;
  for (k = 0; k < n; ++k) free(desc[k]);
  free(desc);
  return rc;
}
