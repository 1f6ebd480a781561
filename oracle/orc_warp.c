/*
 * orc_warp.c — plain-C restatement of the reference's cylindrical pre-warp.
 * TEST INFRASTRUCTURE ONLY (see orc_common.h).  Citations relative to
 * the reference's src/.
 */
#include <float.h>
#include "orc_common.h"

typedef struct { double cx, cy; int r; int sizefactor; } cylproj;

/* stitch/warp.cc:70-75 CylinderWarper::get_projector */
static cylproj get_projector(int w, int h, double h_factor, const pano_params* P) {
  cylproj c;
  c.r = (int)(hypot((double)w, (double)h) * (P->focal_length / 43.266));
  c.cx = w / 2;
  c.cy = h / 2 * h_factor;
  c.sizefactor = c.r;
  return c;
}

/* stitch/warp.cc:13-17 proj */
static void proj(const cylproj* c, double px, double py, double* ox, double* oy) {
  *ox = atan((px - c->cx) / c->r);
  *oy = (py - c->cy) / hypot(px - c->cx, (double)c->r);
}

/* stitch/warp.cc:19-23 proj_r */
static void proj_r(const cylproj* c, double px, double py, double* ox, double* oy) {
  *ox = c->r * tan(px) + c->cx;
  *oy = py * c->r / cos(px) + c->cy;
}

/* stitch/warp.cc:46-67 project(Shape2D&, pts) */
static void project_shape(const cylproj* c, int* w, int* h, double* kpts, int nk, double* offx, double* offy) {
  double minx = DBL_MAX, miny = DBL_MAX, maxx = 0, maxy = 0, rsx, rsy;
  int i, j, sx, sy;
  for (i = 0; i < *h; ++i)
    for (j = 0; j < *w; ++j) {
      double x, y;
      proj(c, j, i, &x, &y);
      if (x < minx) minx = x;
      if (y < miny) miny = y;
      if (maxx < x) maxx = x;
      if (maxy < y) maxy = y;
    }
  maxx = maxx * c->sizefactor; maxy = maxy * c->sizefactor;
  minx = minx * c->sizefactor; miny = miny * c->sizefactor;
  rsx = maxx - minx; rsy = maxy - miny;
  *offx = minx * (-1); *offy = miny * (-1);
  sx = (int)rsx; sy = (int)rsy;
  for (i = 0; i < nk; ++i) {
    double x, y;
    proj(c, kpts[2 * i] + *w / 2, kpts[2 * i + 1] + *h / 2, &x, &y);
    x = x * c->sizefactor + *offx;
    y = y * c->sizefactor + *offy;
    x -= sx / 2;
    y -= sy / 2;
    kpts[2 * i] = x; kpts[2 * i + 1] = y;
  }
  *w = sx; *h = sy;
}

int orc_cyl_warp_shape(int w, int h, double h_factor, const pano_params* P,
                       int* ow, int* oh, double* offx, double* offy) {
  cylproj c = get_projector(w, h, h_factor, P);
  *ow = w; *oh = h;
  project_shape(&c, ow, oh, NULL, 0, offx, offy);
  return 0;
}

/* stitch/warp.cc:25-44 project(img, pts) */
int orc_cyl_warp(const float* rgb, int w, int h, double h_factor, const pano_params* P,
                 float* out, int ow, int oh, double* kpts, int nk) {
  cylproj c = get_projector(w, h, h_factor, P);
  int sw = w, sh = h, i, j;
  double offx, offy, sizefactor_inv;
  project_shape(&c, &sw, &sh, kpts, nk, &offx, &offy);
  if (sw != ow || sh != oh) return -1;
  sizefactor_inv = 1.0 / c.sizefactor;
  for (i = 0; i < oh; ++i)
    for (j = 0; j < ow; ++j) {
      float* p = out + ((size_t)i * ow + j) * 3;
      double x, y;
      float col[3];
      p[0] = p[1] = p[2] = -1.f; /* Color::NO */
      proj_r(&c, (j - offx) * sizefactor_inv, (i - offy) * sizefactor_inv, &x, &y);
      if (ORC_BETWEEN(x, 0, w) && ORC_BETWEEN(y, 0, h)) {
        if (orc_interpolate(rgb, w, h, (float)y, (float)x, col)) { p[0] = col[0]; p[1] = col[1]; p[2] = col[2]; }
      }
    }
  return 0;
}
