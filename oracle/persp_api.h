/*
 * persp_api.h — checker API of cylinder mode's perspective correction, CylinderStitcher::perspective_correction
 * (stitch/cylstitcher.cc:139-180).  TEST INFRASTRUCTURE ONLY.
 *   - oracle/liboracle_persp.so              orc_ : plain-C restatement of the correction pass (oracle/orc_persp.c)
 *   - oracle/_ref/libopenpano_ref_persp.so   ref_ : the reference's own perspective_correction, reached through a
 *                                                   test subclass of CylinderStitcher (oracle/refshim/ref_persp.cc)
 * Both are built by oracle/cyl_sweep.mk.
 */
#ifndef PERSP_API_H
#define PERSP_API_H

#include "../include/pano_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The correction pass on a w×h×3 f32 mosaic: LinearBlender of the one image over ROI (0, 0)–(w, h) with the map
 * inv.trans2d(c), LAZY_READ / ORDERED_INPUT from lazy_read / ordered_input.  out: w×h×3 f32.  0 on success. */
int orc_persp_correct(const float* mosaic, int w, int h, const double inv[9], int lazy_read, int ordered_input,
                      float* out);

/* The reference's perspective_correction on the same mosaic, under LAZY_READ / ORDERED_INPUT as given, with the
 * correction homography handed over: its call of getPerspectiveTransform on the four corners returns inv (the
 * caller's host solve, as the engine takes it).  out: w×h×3 f32.  0 on success.  Not thread-safe (the
 * reference's config globals and the hand-over). */
int ref_persp_correction(const float* mosaic, int w, int h, const double inv[9], int lazy_read, int ordered_input,
                         float* out);
/* The two point sets the reference's perspective_correction hands to getPerspectiveTransform for a w×h mosaic and
 * the bundle of three images (first, identity, last) of shapes {w, h} x 3 (the warped shapes), the first and last
 * components' homo (3×3, row-major), proj_range.min = (proj_min_x, proj_min_y) and the flat projection: corners
 * and targets, 4 points (x, y) each.  0 on success.  Not thread-safe. */
int ref_persp_points(const int shapes[6], const double first_homo[9], const double last_homo[9], double proj_min_x,
                     double proj_min_y, int w, int h, double corners[8], double targets[8]);

#ifdef __cplusplus
}
#endif
#endif
