/*
 * orc_planet.c — plain-C restatement of the reference's little-planet view, planet() (main.cc:294-331,
 * the `planet` sub-command at :352-353).  TEST INFRASTRUCTURE ONLY (see orc_common.h).  Citations
 * relative to the reference's src/.  Pinned against the reference's own planet() by
 * tests/test_oracle_planet.py (ref_planet, oracle/refshim/ref_planet.cc).
 */
#include "orc_common.h"
#include "planet_api.h"

int orc_planet(const float* img, int w, int h, float* out) {
  const int OUTSIZE = ORC_PLANET_SIZE, center = OUTSIZE / 2;       /* :297 */
  int i, j;
  size_t k;
  if (w < 1 || h < 1) return -1;
  for (k = 0; k < (size_t)OUTSIZE * OUTSIZE * 3; ++k) out[k] = -1.0f;   /* :298-299 fill(ret, Color::NO) */
  for (i = 0; i < OUTSIZE; ++i)
    for (j = 0; j < OUTSIZE; ++j) {
      double dist = hypot((double)(center - i), (double)(center - j));  /* :302 */
      double theta;
      float c[3];
      if (dist >= center || dist == 0) continue;                        /* :303 */
      dist = dist / center;                                             /* :304 */
      dist = h - dist * h;                                              /* :306 */
      if (j == center) {                                                /* :308-319 */
        if (i < center) theta = M_PI / 2;
        else theta = 3 * M_PI / 2;
      } else {
        theta = atan((double)(center - i) / (center - j));
        if (theta < 0) theta += M_PI;
        if ((theta == 0) && (j > center)) theta += M_PI;
        if (center < i) theta += M_PI;
      }
      theta = theta / (M_PI * 2) * w;                                   /* :323 */
      if ((double)h - 1 < dist) dist = (double)h - 1;                   /* :325 update_min, lib/utils.hh:50-55 */
      if (orc_interpolate(img, w, h, (float)dist, (float)theta, c)) {   /* :326-328; Color::NO writes -1 */
        float* p = out + ((size_t)i * OUTSIZE + j) * 3;
        p[0] = c[0]; p[1] = c[1]; p[2] = c[2];
      }
    }
  return 0;
}
