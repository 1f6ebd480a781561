/*
 * ba_step_api.h — checker API for one LM iteration's per-point work of bundle adjustment beyond the
 * Jacobian (stitch/incremental_bundle_adjuster.cc:171-220, :237-238).  TEST INFRASTRUCTURE ONLY.
 *   - oracle/liboracle_ba_step.so          orc_ : plain-C restatement (oracle/orc_ba_step.c)
 *   - oracle/_ref/libopenpano_ref_ba_step.so ref_ : the reference's own TU (oracle/refshim/ref_ba_step.cc)
 * Both are built by oracle/ba_step.mk.  Pairs use orc_ba_pair of oracle_api.h; its m is ignored here.
 */
#ifndef BA_STEP_API_H
#define BA_STEP_API_H
#include "oracle_api.h"

#ifdef __cplusplus
extern "C" {
#endif

/* calcError + update_stats from the per-pair Hto_to_from (9 doubles each, an input like the Jacobian's
 * matrices) and pts (4 doubles per match {to.x, to.y, from.x, from.y}) -> residuals (2 per match), avg, max. */
int orc_ba_error(int n_pair, const orc_ba_pair* pairs, const double* hto, const double* pts, double* residuals,
                 double* avg, double* max);
/* b = J^T * residuals (6 n_cam) from the compact rows of orc_ba_jacobian. */
int orc_ba_jtr(int n_cam, int n_pair, const orc_ba_pair* pairs, const double* j_rows, const double* residuals,
               double* b);
/* The reference's own calcError(state) for the cameras (12 doubles each {focal, ppx, ppy, R[9]}); also the
 * per-pair (c_from.K() * c_from.R) * (c_to.Rinv() * c_to.K().inverse()) made by the reference's operations
 * (hto, 9 per pair). */
int ref_ba_error(int n_cam, const double* cams, int n_pair, const orc_ba_pair* pairs, const double* pts,
                 double* residuals, double* avg, double* max, double* hto);
/* calcJacobianSymbolic(state) for the cameras, then the TU's J.transpose() * Map<const VectorXd>(residuals)
 * with the given residuals (2 per match). */
int ref_ba_jtr(int n_cam, const double* cams, int n_pair, const orc_ba_pair* pairs, const double* pts,
               const double* residuals, double* b);

#ifdef __cplusplus
}
#endif
#endif
