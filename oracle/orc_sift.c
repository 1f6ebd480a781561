/*
 * orc_sift.c — plain-C restatement of the reference's SIFT chain.
 * TEST INFRASTRUCTURE ONLY (see orc_common.h for who may load it and for the
 * parity-pinning status).  Citations are relative to the reference's src/.
 */
#include <stdio.h>
#include "orc_common.h"
#include "small_linalg.h"

#define MAX_OCT 16
#define MAX_SCALE 16

typedef struct {
  int w, h;
  float* data[MAX_SCALE]; /* gaussian levels 0..nscale-1 */
  float* mag[MAX_SCALE];  /* 1..nscale-1 */
  float* ort[MAX_SCALE];
  float* dog[MAX_SCALE];  /* 0..nscale-2 */
} orc_octave;

typedef struct { pano_sspoint* v; int n, cap; } pt_list;

struct orc_sift {
  int in_w, in_h;
  int w0, h0;
  int noct, nscale;
  float* working; /* h0*w0*3 */
  orc_octave oct[MAX_OCT];
  pt_list raw, refined, oriented;
  float* desc;   /* n*128 */
  double* coor;  /* n*2, detect_feature output coordinates */
  pano_params P;
};

static void pt_push(pt_list* l, const pano_sspoint* p) {
  if (l->n == l->cap) {
    l->cap = l->cap ? l->cap * 2 : 1024;
    l->v = (pano_sspoint*)realloc(l->v, sizeof(pano_sspoint) * (size_t)l->cap);
  }
  l->v[l->n++] = *p;
}

/* lib/imgproc.cc:22-80 resize_bilinear (3-channel) */
static void resize_bilinear3(const float* src, int sw, int sh, float* dst, int dw, int dh) {
  int* tabsx = (int*)malloc(sizeof(int) * (size_t)dh);
  int* tabsy = (int*)malloc(sizeof(int) * (size_t)dw);
  float* tabrx = (float*)malloc(sizeof(float) * (size_t)dh);
  float* tabry = (float*)malloc(sizeof(float) * (size_t)dw);
  const float fx = (float)dh / sh;
  const float fy = (float)dw / sw;
  const float ifx = 1.f / fx;
  const float ify = 1.f / fy;
  int dx, dy, c;
  for (dx = 0; dx < dh; ++dx) {
    float rx = (dx + 0.5f) * ifx - 0.5f;
    int sx = (int)floor(rx);
    rx -= sx;
    if (sx < 0) { sx = 0; rx = 0; }
    else if (sx + 1 >= sh) { sx = sh - 2; rx = 1; }
    tabsx[dx] = sx; tabrx[dx] = rx;
  }
  for (dy = 0; dy < dw; ++dy) {
    float ry = (dy + 0.5f) * ify - 0.5f;
    int sy = (int)floor(ry);
    ry -= sy;
    if (sy < 0) { sy = 0; ry = 0; }
    else if (sy + 1 >= sw) { sy = sw - 2; ry = 1; }
    tabsy[dy] = sy; tabry[dy] = ry;
  }
  for (dx = 0; dx < dh; ++dx) {
    const float* p0 = src + (size_t)tabsx[dx] * sw * 3;
    const float* p1 = src + (size_t)(tabsx[dx] + 1) * sw * 3;
    float* pdst = dst + (size_t)dx * dw * 3;
    float rx = tabrx[dx], irx = 1.0f - rx;
    for (dy = 0; dy < dw; ++dy) {
      const float* pc00 = p0 + (tabsy[dy] + 0) * 3;
      const float* pc01 = p0 + (tabsy[dy] + 1) * 3;
      const float* pc10 = p1 + (tabsy[dy] + 0) * 3;
      const float* pc11 = p1 + (tabsy[dy] + 1) * 3;
      float ry = tabry[dy], iry = 1.0f - ry;
      for (c = 0; c < 3; ++c)
        pdst[dy * 3 + c] = rx * (pc11[c] * ry + pc10[c] * iry) + irx * (pc01[c] * ry + pc00[c] * iry);
    }
  }
  free(tabsx); free(tabsy); free(tabrx); free(tabry);
}

/* feature/dog.cc:22-37 fast_atan */
static float fast_atan(float y, float x) {
  float absx = fabsf(x), absy = fabsf(y);
  float m = absx > absy ? absx : absy; /* std::max(absx, absy) */
  float a, s, r;
  if (m < ORC_EPS) return (float)-M_PI;
  a = (absy < absx ? absy : absx) / m; /* std::min(absx, absy) / m */
  s = a * a;
  r = (float)(((-0.0464964749 * s + 0.15931422) * s - 0.327622764) * s * a + a);
  if (absy > absx) r = (float)(M_PI_2 - r);
  if (x < 0) r = (float)(M_PI - r);
  if (y < 0) r = -r;
  return r;
}

/* feature/dog.cc:60-94 cal_mag_ort */
static void cal_mag_ort(const float* img, int w, int h, float* mag, float* ort) {
  int x, y;
  for (y = 0; y < h; ++y) {
    float* mrow = mag + (size_t)y * w;
    float* orow = ort + (size_t)y * w;
    const float* row = img + (size_t)y * w;
    const float* plus = row + w;
    const float* minus = row - w;
    mrow[0] = 0; orow[0] = (float)M_PI;
    for (x = 1; x < w - 1; ++x) {
      if (ORC_BETWEEN(y, 1, h - 1)) {
        float dy = plus[x] - minus[x], dx = row[x + 1] - row[x - 1];
        mrow[x] = hypotf(dx, dy);
        orow[x] = (float)(fast_atan(dy, dx) + M_PI);
      } else {
        mrow[x] = 0; orow[x] = (float)M_PI;
      }
    }
    mrow[w - 1] = 0; orow[w - 1] = (float)M_PI;
  }
}

/* feature/dog.cc:42-58 GaussianPyramid ctor + dog.cc:116-143 DOGSpace */
static void build_octave(orc_octave* o, const float* rgb, int w, int h, const pano_params* P) {
  size_t n = (size_t)w * h, i;
  int s, ns = P->num_scale;
  float sigma = P->gauss_sigma;
  o->w = w; o->h = h;
  memset(o->data, 0, sizeof(o->data)); memset(o->mag, 0, sizeof(o->mag));
  memset(o->ort, 0, sizeof(o->ort)); memset(o->dog, 0, sizeof(o->dog));
  o->data[0] = (float*)malloc(sizeof(float) * n);
  for (i = 0; i < n; ++i) /* lib/imgproc.cc:237-249 rgb2grey */
    o->data[0][i] = (rgb[i * 3] + rgb[i * 3 + 1] + rgb[i * 3 + 2]) / 3.f;
  for (s = 1; s < ns; ++s) { /* gaussian.hh:93-107: sigma_k = sigma * factor^k, float product */
    float kernel[128];
    int kw = orc_gauss_kernel(sigma, P->gauss_window_factor, kernel);
    o->data[s] = (float*)malloc(sizeof(float) * n);
    orc_blur(o->data[0], o->data[s], w, h, 1, kernel, kw); /* always from level 0 (dog.cc:55) */
    o->mag[s] = (float*)malloc(sizeof(float) * n);
    o->ort[s] = (float*)malloc(sizeof(float) * n);
    cal_mag_ort(o->data[s], w, h, o->mag[s], o->ort[s]);
    sigma *= P->scale_factor;
  }
  for (s = 0; s < ns - 1; ++s) {
    o->dog[s] = (float*)malloc(sizeof(float) * n);
    for (i = 0; i < n; ++i) o->dog[s][i] = fabsf(o->data[s][i] - o->data[s + 1][i]);
  }
}

/* feature/extrema.cc:170-216 get_local_raw_extrema's predicate */
static int is_extrema(const orc_octave* o, int scale, int r, int c, const pano_params* P) {
  const float* now = o->dog[scale];
  int w = o->w, di, dj, ds, mx = 1, mn = 1;
  float center = now[(size_t)r * w + c], cmp1, cmp2;
  if (center < P->pre_color_thres) return 0;
  cmp1 = center - P->judge_extrema_diff_thres;
  cmp2 = center + P->judge_extrema_diff_thres;
  for (di = -1; di < 2; ++di)
    for (dj = -1; dj < 2; ++dj) {
      float v;
      if (!di && !dj) continue;
      v = now[(size_t)(r + di) * w + c + dj];
      if (v >= cmp1) mx = 0;
      if (v <= cmp2) mn = 0;
      if (!mx && !mn) return 0;
    }
  for (ds = -1; ds < 2; ds += 2) {
    const float* mat = o->dog[scale + ds];
    for (di = -1; di < 2; ++di)
      for (dj = -1; dj < 2; ++dj) {
        float v = mat[(size_t)(r + di) * w + c + dj];
        if (v >= cmp1) mx = 0;
        if (v <= cmp2) mn = 0;
        if (!mx && !mn) return 0;
      }
  }
  return 1;
}

/* feature/extrema.cc:108-150 calc_kp_offset_iter */
static void kp_offset_iter(const orc_octave* o, int x, int y, int s, double offset[3], double delta[3]) {
  int w = o->w;
#define D(xx, yy, ss) (o->dog[ss][(size_t)(yy) * w + (xx)])
  float val = D(x, y, s);
  double dxx, dyy, dss, dxy, dys, dsx, m[9], inv[9];
  delta[0] = (D(x + 1, y, s) - D(x - 1, y, s)) / 2;
  delta[1] = (D(x, y + 1, s) - D(x, y - 1, s)) / 2;
  delta[2] = (D(x, y, s + 1) - D(x, y, s - 1)) / 2;
  dxx = D(x + 1, y, s) + D(x - 1, y, s) - val - val;
  dyy = D(x, y + 1, s) + D(x, y - 1, s) - val - val;
  dss = D(x, y, s + 1) + D(x, y, s - 1) - val - val;
  dxy = (D(x + 1, y + 1, s) - D(x + 1, y - 1, s) - D(x - 1, y + 1, s) + D(x - 1, y - 1, s)) / 4;
  dys = (D(x, y + 1, s + 1) - D(x, y - 1, s + 1) - D(x, y + 1, s - 1) + D(x, y - 1, s - 1)) / 4;
  dsx = (D(x + 1, y, s + 1) - D(x - 1, y, s + 1) - D(x + 1, y, s - 1) + D(x - 1, y, s - 1)) / 4;
#undef D
  m[0] = dxx; m[4] = dyy; m[8] = dss;
  m[1] = m[3] = dxy; m[2] = m[6] = dsx; m[5] = m[7] = dys;
  if (!orc_lu3_inverse(m, inv)) orc_sym3_pinv(m, inv);
  {
    int i;
    for (i = 0; i < 3; ++i) {
      double acc = inv[i * 3] * delta[0];
      acc += inv[i * 3 + 1] * delta[1];
      acc += inv[i * 3 + 2] * delta[2];
      offset[i] = acc;
    }
  }
}

/* feature/extrema.cc:63-106 calc_kp_offset */
static int calc_kp_offset(const orc_octave* o, pano_sspoint* sp, const pano_params* P) {
  int w = o->w, h = o->h, nscale = P->num_scale;
  int nowx = sp->x, nowy = sp->y, nows = sp->scale_id, niter = 0;
  double offset[3] = {0, 0, 0}, delta[3] = {0, 0, 0}, dextr;
  for (; niter < P->calc_offset_depth; ++niter) {
    double am;
    if (!ORC_BETWEEN(nowx, 1, w - 1) || !ORC_BETWEEN(nowy, 1, h - 1) || !ORC_BETWEEN(nows, 1, nscale - 2))
      return 0;
    kp_offset_iter(o, nowx, nowy, nows, offset, delta);
    am = fmax(fabs(offset[0]), fmax(fabs(offset[1]), fabs(offset[2])));
    if (am < P->offset_thres) break;
    nowx = (int)(nowx + round(offset[0]));
    nowy = (int)(nowy + round(offset[1]));
    nows = (int)(nows + round(offset[2]));
  }
  if (niter == P->calc_offset_depth) return 0;
  dextr = offset[0] * delta[0] + offset[1] * delta[1] + offset[2] * delta[2];
  dextr = o->dog[nows][(size_t)nowy * w + nowx] + dextr / 2;
  if (dextr < P->contrast_thres) return 0;
  sp->x = nowx; sp->y = nowy; sp->scale_id = nows;
  sp->scale_factor = (float)(P->gauss_sigma * pow((double)P->scale_factor, ((double)nows + offset[2]) / nscale));
  sp->real_x = ((double)nowx + offset[0]) / w;
  sp->real_y = ((double)nowy + offset[1]) / h;
  return 1;
}

/* feature/extrema.cc:152-168 is_edge_response */
static int is_edge_response(const float* img, int w, int x, int y, const pano_params* P) {
  float val = img[(size_t)y * w + x];
  float dxx = img[(size_t)y * w + x + 1] + img[(size_t)y * w + x - 1] - val - val;
  float dyy = img[(size_t)(y + 1) * w + x] + img[(size_t)(y - 1) * w + x] - val - val;
  float dxy = (img[(size_t)(y + 1) * w + x + 1] + img[(size_t)(y - 1) * w + x - 1] -
               img[(size_t)(y + 1) * w + x - 1] - img[(size_t)(y - 1) * w + x + 1]) / 4;
  float det = dxx * dyy - dxy * dxy, tr2;
  if (det <= 0) return 1;
  tr2 = orc_sqrf(dxx + dyy);
  if (tr2 / det < orc_sqrf(P->edge_ratio + 1) / P->edge_ratio) return 0;
  return 1;
}

#define ORI_BINS 36
/* feature/orientation.cc:34-100 calc_dir; returns number of peaks, dirs[<=36] */
static int calc_dir(const orc_octave* o, const pano_sspoint* p, const pano_params* P, float* dirs) {
  const float halfipi = (float)(0.5f / M_PI);
  const float* ort_img = o->ort[p->scale_id];
  const float* mag_img = o->mag[p->scale_id];
  float gauss_weight_sigma = p->scale_factor * 1.5f; /* ORI_WINDOW_FACTOR, config.hh:74 */
  int rad = (int)roundf(p->scale_factor * P->ori_radius);
  float exp_denom = 2 * orc_sqrf(gauss_weight_sigma);
  float hist[ORI_BINS], maxbin = 0, thres;
  int xx, yy, i, K, n = 0;
  memset(hist, 0, sizeof(hist));
  for (xx = -rad; xx < rad; xx++) {
    int newx = p->x + xx;
    if (!ORC_BETWEEN(newx, 1, o->w - 1)) continue;
    for (yy = -rad; yy < rad; yy++) {
      int newy = p->y + yy, bin;
      float orient, weight;
      if (!ORC_BETWEEN(newy, 1, o->h - 1)) continue;
      if (orc_sqrf((float)xx) + orc_sqrf((float)yy) > orc_sqrf((float)rad)) continue;
      orient = ort_img[(size_t)newy * o->w + newx];
      bin = (int)roundf(ORI_BINS * halfipi * orient);
      if (bin == ORI_BINS) bin = 0;
      weight = expf(-(orc_sqrf((float)xx) + orc_sqrf((float)yy)) / exp_denom);
      hist[bin] += weight * mag_img[(size_t)newy * o->w + newx];
    }
  }
  for (K = P->ori_hist_smooth_count; K--;)
    for (i = 0; i < ORI_BINS; ++i) { /* in place, sequential */
      float prev = hist[i == 0 ? ORI_BINS - 1 : i - 1];
      float next = hist[i == ORI_BINS - 1 ? 0 : i + 1];
      hist[i] = (float)(hist[i] * 0.5 + (prev + next) * 0.25);
    }
  for (i = 0; i < ORI_BINS; ++i) if (maxbin < hist[i]) maxbin = hist[i];
  thres = maxbin * 0.8f; /* ORI_HIST_PEAK_RATIO, config.hh:76 */
  for (i = 0; i < ORI_BINS; ++i) {
    float prev = hist[i == 0 ? ORI_BINS - 1 : i - 1];
    float next = hist[i == ORI_BINS - 1 ? 0 : i + 1];
    if (hist[i] > thres && hist[i] > (prev < next ? next : prev)) {
      double newbin = (float)i - 0.5 + (hist[i] - prev) / (prev + next - 2 * hist[i]);
      if (newbin < 0) newbin += ORI_BINS;
      else if (newbin >= ORI_BINS) newbin -= ORI_BINS;
      dirs[n++] = (float)(newbin / ORI_BINS * 2 * M_PI);
    }
  }
  return n;
}

/* feature/sift.cc:48-67 trilinear_interpolate */
static void trilinear(float xbin, float ybin, float hbin, float weight, float hist[16][8]) {
  int ybinf = (int)floorf(ybin), xbinf = (int)floorf(xbin), hbinf = (int)floorf(hbin);
  float ybind = ybin - ybinf, xbind = xbin - xbinf, hbind = hbin - hbinf;
  int dy, dx;
  for (dy = 0; dy < 2; ++dy)
    if (ORC_BETWEEN(ybinf + dy, 0, 4)) {
      float w_y = weight * (dy ? ybind : 1 - ybind);
      for (dx = 0; dx < 2; ++dx)
        if (ORC_BETWEEN(xbinf + dx, 0, 4)) {
          float w_x = w_y * (dx ? xbind : 1 - xbind);
          int idx = (ybinf + dy) * 4 + (xbinf + dx);
          hist[idx][hbinf % 8] += w_x * (1 - hbind);
          hist[idx][(hbinf + 1) % 8] += w_x * hbind;
        }
    }
}

/* feature/sift.cc:87-152 calc_descriptor + :15-46 hist_to_descriptor (RootSIFT) */
static void calc_descriptor(const orc_octave* o, const pano_sspoint* p, const pano_params* P, float* out) {
  const float pi2 = (float)(2 * M_PI);
  const float nbin_per_rad = 8 / pi2;
  int w = o->w, h = o->h;
  const float* mag_img = o->mag[p->scale_id];
  const float* ort_img = o->ort[p->scale_id];
  float ort = p->dir;
  float hist_w = p->scale_factor * P->desc_hist_scale_factor;
  float exp_denom = 2 * orc_sqrf(4);
  int radius = (int)round(M_SQRT1_2 * hist_w * (4 + 1));
  float hist[16][8], cosort = cosf(ort), sinort = sinf(ort), sum;
  float* hf = &hist[0][0];
  int xx, yy, i;
  memset(hist, 0, sizeof(hist));
  for (xx = -radius; xx <= radius; xx++) {
    int nowx = p->x + xx;
    if (!ORC_BETWEEN(nowx, 1, w - 1)) continue;
    for (yy = -radius; yy <= radius; yy++) {
      int nowy = p->y + yy;
      float y_rot, x_rot, ybin, xbin, now_mag, now_ort, weight, hist_bin;
      if (!ORC_BETWEEN(nowy, 1, h - 1)) continue;
      if (orc_sqrf((float)xx) + orc_sqrf((float)yy) > orc_sqrf((float)radius)) continue;
      y_rot = (-xx * sinort + yy * cosort) / hist_w;
      x_rot = (xx * cosort + yy * sinort) / hist_w;
      ybin = (float)(y_rot + 4 / 2 - 0.5);
      xbin = (float)(x_rot + 4 / 2 - 0.5);
      if (!ORC_BETWEEN(ybin, -1, 4) || !ORC_BETWEEN(xbin, -1, 4)) continue;
      now_mag = mag_img[(size_t)nowy * w + nowx];
      now_ort = ort_img[(size_t)nowy * w + nowx];
      weight = expf(-(orc_sqrf(x_rot) + orc_sqrf(y_rot)) / exp_denom);
      weight = weight * now_mag;
      now_ort -= ort;
      if (now_ort < 0) now_ort += pi2;
      if (now_ort > pi2) now_ort -= pi2;
      hist_bin = now_ort * nbin_per_rad;
      trilinear(xbin, ybin, hist_bin, weight, hist);
    }
  }
  sum = 0;
  for (i = 0; i < 128; ++i) sum += hf[i];
  for (i = 0; i < 128; ++i) out[i] = hf[i] / sum;
  for (i = 0; i < 128; ++i) out[i] = sqrtf(out[i]) * P->desc_int_factor;
}

/* feature/feature.cc:31-47 do_detect_feature + :20-28 detect_feature */
orc_sift* orc_sift_run(const float* rgb, int w, int h, const pano_params* P) {
  orc_sift* s = (orc_sift*)calloc(1, sizeof(orc_sift));
  float ratio = P->sift_working_size * 2.0f / (w + h);
  int o, j, r, c, i;
  s->P = *P; s->in_w = w; s->in_h = h;
  s->noct = P->num_octave; s->nscale = P->num_scale;
  s->h0 = (int)(h * ratio); s->w0 = (int)(w * ratio);
  s->working = (float*)malloc(sizeof(float) * (size_t)s->w0 * s->h0 * 3);
  resize_bilinear3(rgb, w, h, s->working, s->w0, s->h0);
  /* feature/dog.cc:96-114 ScaleSpace: octave i>0 is resized from the WORKING image */
  for (o = 0; o < s->noct; ++o) {
    if (!o) build_octave(&s->oct[0], s->working, s->w0, s->h0, P);
    else {
      float factor = (float)pow((double)P->scale_factor, (double)-o);
      int neww = (int)ceilf(s->w0 * factor), newh = (int)ceilf(s->h0 * factor);
      float* resized = (float*)malloc(sizeof(float) * (size_t)neww * newh * 3);
      resize_bilinear3(s->working, s->w0, s->h0, resized, neww, newh);
      build_octave(&s->oct[o], resized, neww, newh, P);
      free(resized);
    }
  }
  /* feature/extrema.cc:36-61 get_extrema, single-thread order: octave, scale, raster */
  for (o = 0; o < s->noct; ++o)
    for (j = 1; j < s->nscale - 2; ++j) {
      const orc_octave* oc = &s->oct[o];
      for (r = 1; r < oc->h - 1; ++r)
        for (c = 1; c < oc->w - 1; ++c)
          if (is_extrema(oc, j, r, c, P)) {
            pano_sspoint sp;
            memset(&sp, 0, sizeof(sp));
            sp.x = c; sp.y = r; sp.pyr_id = o; sp.scale_id = j;
            pt_push(&s->raw, &sp);
            if (!calc_kp_offset(oc, &sp, P)) continue;
            if (is_edge_response(oc->dog[sp.scale_id], oc->w, sp.x, sp.y, P)) continue;
            pt_push(&s->refined, &sp);
          }
    }
  /* feature/orientation.cc:22-32 work */
  for (i = 0; i < s->refined.n; ++i) {
    float dirs[ORI_BINS];
    int k, nd = calc_dir(&s->oct[s->refined.v[i].pyr_id], &s->refined.v[i], P, dirs);
    for (k = 0; k < nd; ++k) {
      pano_sspoint sp = s->refined.v[i];
      sp.dir = dirs[k];
      pt_push(&s->oriented, &sp);
    }
  }
  /* feature/sift.cc:77-85 get_descriptor; feature.cc:20-28 coordinate shift */
  s->desc = (float*)malloc(sizeof(float) * 128 * (size_t)(s->oriented.n + 1));
  s->coor = (double*)malloc(sizeof(double) * 2 * (size_t)(s->oriented.n + 1));
  for (i = 0; i < s->oriented.n; ++i) {
    const pano_sspoint* p = &s->oriented.v[i];
    calc_descriptor(&s->oct[p->pyr_id], p, P, s->desc + (size_t)128 * i);
    s->coor[2 * i] = (p->real_x - 0.5) * w;
    s->coor[2 * i + 1] = (p->real_y - 0.5) * h;
  }
  return s;
}

void orc_sift_working_size(const orc_sift* s, int* w0, int* h0) { *w0 = s->w0; *h0 = s->h0; }

int orc_sift_octave_size(const orc_sift* s, int o, int* w, int* h) {
  if (o < 0 || o >= s->noct) return -1;
  *w = s->oct[o].w; *h = s->oct[o].h;
  return 0;
}

int orc_sift_plane(const orc_sift* s, int kind, int o, int level, float* out) {
  const float* src = NULL;
  size_t n;
  if (kind == 0) { memcpy(out, s->working, sizeof(float) * (size_t)s->w0 * s->h0 * 3); return 0; }
  if (o < 0 || o >= s->noct) return -1;
  n = (size_t)s->oct[o].w * s->oct[o].h;
  if (kind == 1 && level >= 0 && level < s->nscale) src = s->oct[o].data[level];
  else if (kind == 2 && level >= 0 && level < s->nscale - 1) src = s->oct[o].dog[level];
  else if (kind == 3 && level >= 1 && level < s->nscale) src = s->oct[o].mag[level];
  else if (kind == 4 && level >= 1 && level < s->nscale) src = s->oct[o].ort[level];
  if (!src) return -1;
  memcpy(out, src, sizeof(float) * n);
  return 0;
}

int orc_sift_points(const orc_sift* s, int stage, int cap, pano_sspoint* out) {
  const pt_list* l = stage == 0 ? &s->raw : stage == 1 ? &s->refined : &s->oriented;
  int i;
  for (i = 0; i < l->n && i < cap; ++i) out[i] = l->v[i];
  return l->n;
}

int orc_sift_descriptors(const orc_sift* s, int cap, double* coor, float* desc) {
  int n = s->oriented.n, m = n < cap ? n : cap;
  if (coor && m) memcpy(coor, s->coor, sizeof(double) * 2 * (size_t)m);
  if (desc && m) memcpy(desc, s->desc, sizeof(float) * 128 * (size_t)m);
  return n;
}

void orc_sift_free(orc_sift* s) {
  int o, k;
  if (!s) return;
  for (o = 0; o < s->noct; ++o)
    for (k = 0; k < MAX_SCALE; ++k) {
      free(s->oct[o].data[k]); free(s->oct[o].mag[k]); free(s->oct[o].ort[k]); free(s->oct[o].dog[k]);
    }
  free(s->working); free(s->raw.v); free(s->refined.v); free(s->oriented.v);
  free(s->desc); free(s->coor); free(s);
}

int orc_sift_detect(const float* rgb, int w, int h, const pano_params* P, int cap, double* coor, float* desc) {
  orc_sift* s = orc_sift_run(rgb, w, h, P);
  int n = s->oriented.n;
  if (n <= cap) orc_sift_descriptors(s, cap, coor, desc);
  orc_sift_free(s);
  return n <= cap ? n : -1;
}

#ifdef ORC_MT
#include <omp.h>
int orc_num_threads(void) { return omp_get_max_threads(); }
#else
int orc_num_threads(void) { return 1; }
#endif
