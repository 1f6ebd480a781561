/*
 * orc_persp.c — plain-C restatement of cylinder mode's perspective correction pass
 * (stitch/cylstitcher.cc:171-179): a LinearBlender (stitch/blender.cc:24-96) of the one image, the mosaic, over
 * ROI (0, 0)–(w, h) with the map inv.trans2d(c) (stitch/homography.hh:53-76).
 * TEST INFRASTRUCTURE ONLY (see orc_common.h).  Citations relative to the reference's src/.
 */
#include "orc_common.h"
#include "persp_api.h"

/* blender.cc:27-36 GET_COLOR_AND_W for the one image; returns 0 for `continue` */
static int persp_color_and_w(const float* img, int w, int h, const double* d, int i, int j, int ordered_input,
                             float color[3], float* wout) {
  double x = j, y = i, rx, ry, rz, denom, ox, oy;
  float r, c, wt;
  rx = d[0] * x + d[1] * y + d[2] * 1.0; /* Homography::trans of Vec(x, y, 1) */
  ry = d[3] * x + d[4] * y + d[5] * 1.0;
  rz = d[6] * x + d[7] * y + d[8] * 1.0;
  denom = 1.0 / rz; /* trans_normalize */
  ox = rx * denom; oy = ry * denom;
  if (ox < 0 || ox >= w || oy < 0 || oy >= h) return 0; /* blender.hh:39-44 map_coor -> NaN */
  if (isnan(ox)) return 0;                               /* img_coor.isNaN() tests x */
  r = (float)oy; c = (float)ox;
  if (!orc_interpolate(img, w, h, r, c, color)) return 0;
  if (color[0] < 0) return 0;
  wt = (float)(0.5 - fabs(c / w - 0.5));
  if (!ordered_input) wt = (float)(wt * (0.5 - fabs(r / h - 0.5)));
  color[0] *= wt; color[1] *= wt; color[2] *= wt;
  *wout = wt;
  return 1;
}

int orc_persp_correct(const float* img, int w, int h, const double inv[9], int lazy_read, int ordered_input,
                      float* out) {
  int i, j;
  if (!img || !inv || !out || w < 1 || h < 1) return -1;
  /* target_size = ROI max = (w, h); every target pixel lies in the ROI under both range rules (blender.cc:45-46,
   * blender.hh:21-24), and one image means each branch adds at most one c·w to zero */
  for (i = 0; i < h; ++i)
    for (j = 0; j < w; ++j) {
      float color[3] = {0, 0, 0}, wt = 0;
      float* p = out + ((size_t)i * w + j) * 3;
      float isum[3] = {0, 0, 0}, wsum = 0;
      if (persp_color_and_w(img, w, h, inv, i, j, ordered_input, color, &wt)) {
        isum[0] += color[0]; isum[1] += color[1]; isum[2] += color[2];
        wsum += wt;
      }
      if (lazy_read) { /* blender.cc:66-76 */
        if (wsum) { p[0] = isum[0] / wsum; p[1] = isum[1] / wsum; p[2] = isum[2] / wsum; }
        else { p[0] = p[1] = p[2] = -1; }
      } else { /* blender.cc:80-93, Vector::operator/(T p) = *this * (1.0 / p) */
        p[0] = p[1] = p[2] = -1;
        if (wsum > 0) {
          float q = (float)(1.0 / wsum);
          p[0] = isum[0] * q; p[1] = isum[1] * q; p[2] = isum[2] * q;
        }
      }
    }
  return 0;
}
