/*
 * orc_ba.c — plain-C restatement of the per-point part of the reference's symbolic
 * bundle-adjustment Jacobian.  TEST INFRASTRUCTURE ONLY (see orc_common.h).  Citations
 * relative to the reference's src/.
 *
 * stitch/incremental_bundle_adjuster.cc:306-383 (IncrementalBundleAdjuster::
 * calcJacobianSymbolic): per point match the derivatives of the residual w.r.t. the 6
 * parameters of both cameras (two rows of J) and the running sums of J^T J.  The per-pair 3x3
 * products in front of the loop are Eigen calls in the reference (Homography::operator*,
 * inverse; Camera::rotation_to_angle) and are INPUTS here, as they are for the CUDA kernel:
 * the 13 matrices of oracle_api.h's orc_ba_pair, evaluated by the caller.
 * Pinned against the reference's own calcJacobianSymbolic by tests/test_oracle_vs_ref.py
 * (ref_ba_jacobian, oracle/refshim/ref_ba.cc).
 */
#include "orc_common.h"
#include "oracle_api.h"

typedef struct { double x, y, z; } vec3;

static vec3 trans(const double* d, vec3 m) {           /* Homography::trans, homography.hh:52-57 */
  vec3 r;
  r.x = d[0] * m.x + d[1] * m.y + d[2] * m.z;
  r.y = d[3] * m.x + d[4] * m.y + d[5] * m.z;
  r.z = d[6] * m.x + d[7] * m.y + d[8] * m.z;
  return r;
}

static const double dKd[3][9] = {                      /* :84-95 dKdfocal, dKdppx, dKdppy */
    {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0},
    {0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0},
    {0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0}};

int orc_ba_jacobian(int n_cam, int n_pair, const orc_ba_pair* pairs, const double* pts_to, double* j_rows,
                    double* jtj) {
  const size_t N = (size_t)n_cam * 6;
  size_t q;
  int pi, k, i, j;
  for (q = 0; q < N * N; ++q) jtj[q] = 0.0;            /* :281 JtJ.setZero() */
  for (pi = 0; pi < n_pair; ++pi) {
    const orc_ba_pair* pr = &pairs[pi];
    const int pf = pr->from * 6, pt = pr->to * 6;      /* :293-294 param_idx_from / param_idx_to */
    for (k = 0; k < pr->n_match; ++k) {
      const double* to2 = pts_to + 2 * (size_t)(pr->match_begin + k);
      vec3 to = {to2[0], to2[1], 1.0};                 /* trans(Vec2D) -> Vec(x, y, 1) */
      vec3 homo = trans(pr->m[0], to);                 /* :308 */
      float hzf = (float)homo.z;                       /* sqr() is lib/utils.hh:25's float overload */
      double hz_sqr_inv = 1.0 / (hzf * hzf);           /* :309 */
      double hz_inv = 1.0 / homo.z;                    /* :310 */
      double dfx[6], dfy[6], dtx[6], dty[6];
      vec3 dot_u2, dh, ku;
#define DRDV(v, ox, oy) do { dh = (v); \
      (ox) = -dh.x * hz_inv + dh.z * homo.x * hz_sqr_inv; \
      (oy) = -dh.y * hz_inv + dh.z * homo.y * hz_sqr_inv; } while (0)   /* :316-319 */
      dot_u2 = trans(pr->m[1], to);                                     /* :323-324 */
      for (i = 0; i < 3; ++i) DRDV(trans(dKd[i], dot_u2), dfx[i], dfy[i]);          /* :326-330 */
      dot_u2 = trans(pr->m[2], to);                                     /* :332 */
      for (i = 0; i < 3; ++i) DRDV(trans(pr->m[3 + i], dot_u2), dfx[3 + i], dfy[3 + i]);   /* :333-335 */
      ku = trans(pr->m[6], to);
      dot_u2.x = ku.x * -1; dot_u2.y = ku.y * -1; dot_u2.z = ku.z * -1;  /* :339 Vec * (-1) */
      for (i = 0; i < 3; ++i) DRDV(trans(pr->m[7 + i], dot_u2), dtx[i], dty[i]);           /* :341-345 */
      for (i = 0; i < 3; ++i) DRDV(trans(pr->m[10 + i], ku), dtx[3 + i], dty[3 + i]);      /* :348-352 */
#undef DRDV
      if (j_rows) {                                    /* :355-361, compact: the 12 non-zero entries of both rows */
        double* r = j_rows + 24 * (size_t)(pr->match_begin + k);
        for (i = 0; i < 6; ++i) { r[i] = dfx[i]; r[6 + i] = dtx[i]; r[12 + i] = dfy[i]; r[18 + i] = dty[i]; }
      }
      for (i = 0; i < 6; ++i)                          /* :364-369 */
        for (j = 0; j < 6; ++j) {
          size_t i1 = pf + i, i2 = pt + j;
          double val = dfx[i] * dtx[j] + dfy[i] * dty[j];     /* Vec2D::dot, geometry.hh:174 */
          jtj[i1 * N + i2] += val; jtj[i2 * N + i1] += val;
        }
      for (i = 0; i < 6; ++i)                          /* :370-381 */
        for (j = i; j < 6; ++j) {
          size_t i1 = pf + i, i2 = pf + j;
          double val = dfx[i] * dfx[j] + dfy[i] * dfy[j];
          jtj[i1 * N + i2] += val;
          if (i != j) jtj[i2 * N + i1] += val;
          i1 = pt + i; i2 = pt + j;
          val = dtx[i] * dtx[j] + dty[i] * dty[j];
          jtj[i1 * N + i2] += val;
          if (i != j) jtj[i2 * N + i1] += val;
        }
    }
  }
  return 0;
}
