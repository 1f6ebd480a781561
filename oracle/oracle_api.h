/*
 * oracle_api.h — the checker API.  TEST INFRASTRUCTURE ONLY.
 *
 * Two libraries implement this same set of functions:
 *   - oracle/liboracle.so        prefix orc_  : plain-C restatement of the
 *                                               reference algorithm (the orc_ C files)
 *   - oracle/_ref/libopenpano_ref.so prefix ref_: the reference's own
 *                                               translation units compiled from
 *                                               the reference's src/ (refshim/)
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load them.  The product (openpano_b200) never does.
 */
#ifndef ORACLE_API_H
#define ORACLE_API_H
#include "../include/pano_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define ORACLE_DECLARE(P)                                                              \
  typedef struct P##_sift P##_sift;                                                    \
  /* runs the whole SIFT chain on one image, keeps every intermediate */              \
  P##_sift* P##_sift_run(const float* rgb_hwc, int w, int h, const pano_params* p);    \
  void P##_sift_working_size(const P##_sift* s, int* w0, int* h0);                     \
  int  P##_sift_octave_size(const P##_sift* s, int octave, int* w, int* h);            \
  /* kind: 0 working RGB, 1 gaussian level, 2 |DoG| level, 3 mag, 4 ort */             \
  int  P##_sift_plane(const P##_sift* s, int kind, int octave, int level, float* out); \
  /* stage: 0 raw extrema, 1 refined keypoints, 2 oriented keypoints */                \
  int  P##_sift_points(const P##_sift* s, int stage, int cap, pano_sspoint* out);      \
  int  P##_sift_descriptors(const P##_sift* s, int cap, double* coor_xy, float* desc); \
  void P##_sift_free(P##_sift* s);                                                     \
  /* detect_feature only (no intermediates kept): returns count, -1 if > cap */        \
  int  P##_sift_detect(const float* rgb_hwc, int w, int h, const pano_params* p,       \
                       int cap, double* coor_xy, float* desc);                         \
  /* FeatureMatcher::match */                                                          \
  int  P##_match(const float* a, int n, const float* b, int m, const pano_params* p,   \
                 int* pairs_out, int* n_pairs_out);                                    \
  int  P##_cyl_warp_shape(int w, int h, double h_factor, const pano_params* p,         \
                          int* out_w, int* out_h, double* off_x, double* off_y);       \
  int  P##_cyl_warp(const float* rgb_hwc, int w, int h, double h_factor,               \
                    const pano_params* p, float* out_hwc, int out_w, int out_h,        \
                    double* kpts_xy, int n_kpts);                                      \
  int  P##_blend(int n, const pano_blend_image* imgs, const pano_blend_geom* g,        \
                 int bands, const pano_params* p, float* out_hwc, int out_w, int out_h);\
  /* One pass of the whole hot path as Stitcher::build() drives it (stitcher.cc:32-64  \
   * minus geometry): calc_feature over n images, n_pairs matches (use_flann: the      \
   * PairWiseMatcher kd-forest path the reference really runs; else the exact         \
   * FeatureMatcher), then the blender.  n_feat[n], n_match[n_pairs], seconds[3]       \
   * (features, match, blend wall time) are outputs. */                               \
  int  P##_hotpath(int n, const float* const* rgb_hwc, const int* w, const int* h,     \
                   int n_pairs, const int* image_ij, int use_flann,                    \
                   const pano_blend_image* bimgs, const pano_blend_geom* g, int bands, \
                   const pano_params* p, float* out_hwc, int out_w, int out_h,         \
                   int* n_feat, int* n_match, double* seconds);                        \
  /* read_img's conversion of decoded 8-bit pixels (imgio.cc:67-90); channels 1|3 */   \
  int  P##_read_img_rgb8(const unsigned char* pix, int w, int h, int channels,         \
                         float* out_hwc);                                              \
  /* crop (imgproc.cc:200-235): out receives the cropped pixels (capacity w*h*3),      \
   * rect = {x0, y0, width, height}; the ref_ build cannot know x0,y0 (crop returns    \
   * only the pixels) and sets them to -1 */                                           \
  int  P##_crop(const float* mat_hwc, int w, int h, int* rect, float* out_hwc);        \
  /* write_rgb's conversion to 8-bit (imgio.cc:98-113) */                              \
  int  P##_write_rgb8(const float* mat_hwc, int w, int h, unsigned char* out);         \
  /* RANSAC inlier scoring (transform_estimate.cc:68-85,132-148): inlier count of every   \
   * hypothesis (9 doubles each, image 2 -> image 1), first hypothesis with the largest   \
   * count, its inlier flags.  kp*_xy: the matched coordinates, 2 doubles per match. */   \
  int  P##_ransac_score(int n_match, const double* kp1_xy, const double* kp2_xy,         \
                        int n_hyp, const double* homos, float inlier_thres,              \
                        int* hyp_counts, int* best_hyp, int* best_count,                 \
                        unsigned char* inlier_flags);                                    \
  /* number of host threads the library will use (1 for the scalar port) */            \
  int  P##_num_threads(void);

ORACLE_DECLARE(orc)
ORACLE_DECLARE(ref)

/* ---- bundle-adjustment Jacobian (SURVEY.md 8f.4; stitch/incremental_bundle_adjuster.cc:276-385).
 * The restatement works from the 13 per-pair matrices the CUDA entry point takes (same layout as
 * pano_ba_pair, include/pano_b200.h); the reference build works from cameras through the reference's
 * own calcJacobianSymbolic and also evaluates the per-pair matrices with the reference's own
 * Homography / Camera operations. */
typedef struct orc_ba_pair {
  int from, to, match_begin, n_match;
  double m[13][9];
} orc_ba_pair;
int orc_ba_jacobian(int n_cam, int n_pair, const orc_ba_pair* pairs, const double* pts_to,
                    double* j_rows /* 24 per match, may be NULL */, double* jtj /* (6 n_cam)^2 */);
/* cams: 12 doubles per camera {focal, ppx, ppy, R[9]}; pairs: from/to camera slots and match ranges
 * (m is written by ref_ba_pair_mats, ignored by ref_ba_jacobian); pts: 4 doubles per match
 * {to.x, to.y, from.x, from.y}. */
int ref_ba_pair_mats(int n_cam, const double* cams, int n_pair, orc_ba_pair* pairs);
int ref_ba_jacobian(int n_cam, const double* cams, int n_pair, const orc_ba_pair* pairs, const double* pts,
                    double* j_rows, double* jtj);

#ifdef __cplusplus
}
#endif
#endif
