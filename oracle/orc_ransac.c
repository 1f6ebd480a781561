/*
 * orc_ransac.c — plain-C restatement of the RANSAC inlier scoring of the reference.
 * TEST INFRASTRUCTURE ONLY (see orc_common.h).  Citations relative to the reference's src/.
 *
 * stitch/transform_estimate.cc:132-148 TransformEstimation::get_inliers and the selection
 * loop of get_transform (:68-85): for every hypothesis (a Homography from image 2 to image 1)
 * count the matches whose transferred point lies within the inlier distance; the FIRST
 * hypothesis with the largest count wins (update_max is a strict <, lib/utils.hh:58-63).
 * Hypothesis generation (random sampling + DLT, :89-130) is host geometry outside the path.
 *
 * One step is unpinned against the real dependency: `f2_homo_coor.prod(trans^T)` is an Eigen
 * product in the reference (lib/matrix.cc, Eigen absent here); the stand-in sums the three
 * terms in index order in double, which is what this file and the CUDA kernel do as well.
 */
#include "orc_common.h"

static int inlier(const double* h, double x2, double y2, double x1, double y1, float inlier_dist) {
  double p[3], idenom, dx, dy, dist;
  int j;
  for (j = 0; j < 3; ++j) { /* row [x2, y2, 1] times trans^T, Matrix::prod order */
    double acc = x2 * h[3 * j];
    acc += y2 * h[3 * j + 1];
    acc += 1.0 * h[3 * j + 2];
    p[j] = acc;
  }
  idenom = 1.f / p[2];                       /* transform_estimate.cc:142 */
  dx = p[0] * idenom - x1;
  dy = p[1] * idenom - y1;
  dist = dx * dx + dy * dy;                  /* Vector2D::sqr, geometry.hh:224 */
  return dist < inlier_dist;                 /* float INLIER_DIST promoted to double */
}

int orc_ransac_score(int n_match, const double* kp1_xy, const double* kp2_xy, int n_hyp, const double* homos,
                     float inlier_thres, int* hyp_counts, int* best_hyp, int* best_count, unsigned char* inlier_flags) {
  const float inlier_dist = inlier_thres * inlier_thres;   /* sqr(float), lib/utils.hh:25 */
  int k, i, maxcnt = -1, best = -1;
  for (k = 0; k < n_hyp; ++k) {
    int cnt = 0;
    for (i = 0; i < n_match; ++i)
      cnt += inlier(homos + 9 * (size_t)k, kp2_xy[2 * i], kp2_xy[2 * i + 1], kp1_xy[2 * i], kp1_xy[2 * i + 1], inlier_dist);
    if (hyp_counts) hyp_counts[k] = cnt;
    if (maxcnt < cnt) { maxcnt = cnt; best = k; }
  }
  *best_hyp = best;
  *best_count = best < 0 ? 0 : maxcnt;
  if (inlier_flags)
    for (i = 0; i < n_match; ++i)
      inlier_flags[i] = best < 0 ? 0 : (unsigned char)inlier(homos + 9 * (size_t)best, kp2_xy[2 * i], kp2_xy[2 * i + 1],
                                                             kp1_xy[2 * i], kp1_xy[2 * i + 1], inlier_dist);
  return 0;
}
