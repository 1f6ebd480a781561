/*
 * orc_common.h — shared helpers of the plain-C oracle.  TEST INFRASTRUCTURE ONLY:
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load liboracle.so; the product never does.
 *
 * Parity status: PINNED — every function here is checked bit-for-bit against the
 * reference's own translation units (oracle/_ref/libopenpano_ref.so, built by
 * oracle/Makefile from the reference's src/) in tests/test_oracle_vs_ref.py, and
 * against the fixtures in tests/golden/ that were generated from that library
 * (tests/golden/make_golden.py).  The one step without a reference-side pin is
 * the 3x3 solve (Eigen absent; see small_linalg.h).
 *
 * Build: gcc -O2 -ffp-contract=off -msse3 (no FMA contraction: SURVEY.md §8c).
 */
#ifndef ORC_COMMON_H
#define ORC_COMMON_H
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "oracle_api.h"

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif
#ifndef M_PI_2
#define M_PI_2 1.57079632679489661923
#endif
#ifndef M_SQRT1_2
#define M_SQRT1_2 0.70710678118654752440
#endif

/* lib/utils.hh:27  between(a,b,c) == (a >= b) && (a <= c - 1) */
#define ORC_BETWEEN(a, b, c) (((a) >= (b)) && ((a) <= (c) - 1))
/* ORC_MT (liboracle_mt.so, -fopenmp): loops whose iterations write disjoint outputs run
 * on all host threads; each output element is still computed by the same sequential
 * arithmetic, so results are bit-identical to the single-thread build (checked by
 * tests/test_oracle_vs_ref.py::test_oracle_mt_equals_oracle). */
#ifdef ORC_MT
#define ORC_PRAGMA(x) _Pragma(#x)
#define ORC_PAR_FOR(clauses) ORC_PRAGMA(omp parallel for clauses)
#else
#define ORC_PAR_FOR(clauses)
#endif
#define ORC_EPS 1e-6 /* lib/utils.hh:23 (real_t = double) */

static inline float orc_sqrf(float x) { return x * x; } /* lib/utils.hh:26 */

/* lib/imgproc.cc:135-156  interpolate(const Mat32f&, float r, float c).
 * Returns 0 and leaves out untouched for Color::NO. */
static inline int orc_interpolate(const float* img, int w, int h, float r, float c, float out[3]) {
  int fr = (int)floor(r), fc = (int)floor(c);
  const float* p;
  float w00, w10, w11, w01;
  if (fr < 0 || fc < 0 || fc + 1 >= w || fr + 1 >= h) return 0;
  r -= fr; c -= fc;
  w00 = (1 - r) * (1 - c); w10 = r * (1 - c); w11 = r * c; w01 = (1 - r) * c;
  p = img + ((size_t)fr * w + fc) * 3;
  if (*p < 0) return 0;
  out[0] = 0 + p[0] * w00; out[1] = 0 + p[1] * w00; out[2] = 0 + p[2] * w00;
  p = img + ((size_t)(fr + 1) * w + fc) * 3;
  if (*p < 0) return 0;
  out[0] += p[0] * w10; out[1] += p[1] * w10; out[2] += p[2] * w10;
  p = img + ((size_t)(fr + 1) * w + fc + 1) * 3;
  if (*p < 0) return 0;
  out[0] += p[0] * w11; out[1] += p[1] * w11; out[2] += p[2] * w11;
  p = img + ((size_t)fr * w + fc + 1) * 3;
  if (*p < 0) return 0;
  out[0] += p[0] * w01; out[1] += p[1] * w01; out[2] += p[2] * w01;
  return 1;
}

/* feature/gaussian.cc:17-40 GaussCache.  kernel must hold >= 64 floats; returns
 * kw, writes the kw weights (index 0 = tap -center). */
static inline int orc_gauss_kernel(float sigma, int window_factor, float* kernel) {
  int kw = (int)(ceil(0.3 * (sigma / 2 - 1) + 0.8) * window_factor);
  int center, i;
  float exp_coeff, wsum, fac;
  float* k;
  if (kw % 2 == 0) kw++;
  center = kw / 2;
  k = kernel + center;
  k[0] = 1;
  exp_coeff = (float)(-1.0 / (sigma * sigma * 2));
  wsum = 1;
  for (i = 1; i <= center; i++) {
    k[i] = expf((float)(i * i) * exp_coeff);
    wsum += k[i] * 2;
  }
  fac = (float)(1.0 / wsum);
  k[0] = fac;
  for (i = 1; i <= center; i++) { k[i] *= fac; k[-i] = k[i]; }
  return kw;
}

/* feature/gaussian.hh:29-90 GaussianBlur::blur<T>, T = nch interleaved floats
 * (nch=1 for Mat32f, nch=4 for WeightedPixel{Color c; float w}: each channel
 * is blurred independently with the same op order).  Column pass first, then
 * row pass over the column result; replicate border. */
static inline void orc_blur(const float* src, float* dst, int w, int h, int nch,
                            const float* kernel /* kw taps */, int kw) {
  int center = kw / 2;
  int n = (w > h ? w : h) + 2 * center;
  float* line_mem = (float*)malloc(sizeof(float) * (size_t)n);
  float* line = line_mem + center;
  const float* k = kernel + center;
  int i, j, t, ch;
  for (ch = 0; ch < nch; ch++) {
    for (j = 0; j < w; j++) {
      for (i = 0; i < h; i++) line[i] = src[((size_t)i * w + j) * nch + ch];
      for (i = 1; i <= center; i++) line[-i] = line[0];
      for (i = 0; i < center; i++) line[h + i] = line[h - 1];
      for (i = 0; i < h; i++) {
        float tmp = 0;
        for (t = -center; t <= center; t++) tmp += line[i + t] * k[t];
        dst[((size_t)i * w + j) * nch + ch] = tmp;
      }
    }
    for (i = 0; i < h; i++) {
      for (j = 0; j < w; j++) line[j] = dst[((size_t)i * w + j) * nch + ch];
      for (j = 1; j <= center; j++) line[-j] = line[0];
      for (j = 0; j < center; j++) line[w + j] = line[w - 1];
      for (j = 0; j < w; j++) {
        float tmp = 0;
        for (t = -center; t <= center; t++) tmp += line[j + t] * k[t];
        dst[((size_t)i * w + j) * nch + ch] = tmp;
      }
    }
  }
  free(line_mem);
}

#endif
