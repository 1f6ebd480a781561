/*
 * orc_ba_step.c — plain-C restatement of the rest of one LM iteration's per-point work of the
 * reference's bundle adjustment, next to orc_ba.c's Jacobian.  TEST INFRASTRUCTURE ONLY (see
 * orc_common.h).  Citations relative to the reference's src/.
 *
 * stitch/incremental_bundle_adjuster.cc:171-197 (calcError) and :199-220 (ErrorStats::update_stats):
 * the residuals and their statistics; :237-238 (get_param_update): b = J.transpose() * err_vec.
 * Pinned against the reference's own TU by tests/test_oracle_ba_step.py (ref_ba_error / ref_ba_jtr,
 * oracle/refshim/ref_ba_step.cc).
 */
#include "orc_common.h"
#include "ba_step_api.h"

typedef struct { double x, y, z; } vec3;

static vec3 trans(const double* d, vec3 m) {           /* Homography::trans, homography.hh:52-57 */
  vec3 r;
  r.x = d[0] * m.x + d[1] * m.y + d[2] * m.z;
  r.y = d[3] * m.x + d[4] * m.y + d[5] * m.z;
  r.z = d[6] * m.x + d[7] * m.y + d[8] * m.z;
  return r;
}

/* hto: per pair Hto_to_from (:182-183), an INPUT like the Jacobian's matrices.  pts: 4 doubles per match,
 * p.first (to) then p.second (from). */
int orc_ba_error(int n_pair, const orc_ba_pair* pairs, const double* hto, const double* pts, double* residuals,
                 double* avg, double* max) {
  size_t idx = 0, n_res;
  int pi, k;
  double a = 0, m = 0;
  for (pi = 0; pi < n_pair; ++pi) {
    const double* h = hto + 9 * (size_t)pi;
    for (k = 0; k < pairs[pi].n_match; ++k) {
      const double* q = pts + 4 * (size_t)(pairs[pi].match_begin + k);
      vec3 to = {q[0], q[1], 1.0};
      vec3 t = trans(h, to);                           /* trans2d -> trans_normalize, homography.hh:53-64 */
      double denom = 1.0 / t.z;
      residuals[idx] = q[2] - t.x * denom;             /* :190-191 */
      residuals[idx + 1] = q[3] - t.y * denom;
      idx += 2;
    }
  }
  n_res = idx;
  for (idx = 0; idx < n_res; ++idx) {                  /* :213-217 */
    float f = (float)residuals[idx];                   /* error_func: sqr(diff) is lib/utils.hh:25's float overload */
    double e = fabs(residuals[idx]);
    a += (double)(f * f);
    if (m < e) m = e;                                  /* update_max, lib/utils.hh:57-63 */
  }
  a /= (double)n_res;                                  /* :218, 0 / 0 = NaN without matches */
  *avg = sqrt(a);
  *max = m;
  return 0;
}

/* :237-238 b = J.transpose() * err_vec.  Eigen's GEMV order is not pinned; this is the order of the
 * checker build's stand-in (oracle/refshim/eigen_stub/Eigen/Dense: one sequential sum over J's rows per
 * column), over the DENSE rows: the entries outside a match's two cameras are the zeros J.setZero() left
 * (:278), and 0 * r is added like every other product. */
int orc_ba_jtr(int n_cam, int n_pair, const orc_ba_pair* pairs, const double* j_rows, const double* residuals,
               double* b) {
  const int N = 6 * n_cam;
  int col, pi, k;
  for (col = 0; col < N; ++col) {
    double acc = 0;
    for (pi = 0; pi < n_pair; ++pi) {
      const int pf = pairs[pi].from * 6, pt = pairs[pi].to * 6;
      for (k = 0; k < pairs[pi].n_match; ++k) {
        const size_t m = (size_t)(pairs[pi].match_begin + k);
        const double* r = j_rows + 24 * m;
        double jx = 0.0, jy = 0.0, v;
        if (col >= pf && col < pf + 6) { jx = r[col - pf]; jy = r[12 + col - pf]; }
        else if (col >= pt && col < pt + 6) { jx = r[6 + col - pt]; jy = r[18 + col - pt]; }
        v = jx * residuals[2 * m];
        acc += v;
        v = jy * residuals[2 * m + 1];
        acc += v;
      }
    }
    b[col] = acc;
  }
  return 0;
}
