// ref_ba_step.cc — the reference's own calcError / update_stats and J.transpose() * err_vec behind the
// checker API of oracle/ba_step_api.h.  TEST INFRASTRUCTURE ONLY.  Like ref_ba.cc, the reference TU is
// compiled WHERE IT LIES by including it (nothing is copied), which makes the private members callable.
// Built into its own library (oracle/ba_step.mk), linked against libopenpano_ref.so for the rest of the
// reference's classes and the Camera / Homography stand-ins.
#include <vector>
#include <set>
#include <map>
#include <array>
#include <memory>
#include <cmath>
#include <iostream>
#include <sstream>
#include <string>
#include <algorithm>
#include <limits>
#define private public            // calcError, calcJacobianSymbolic, J, match_pairs ... are private members
#define protected public
#include "stitch/incremental_bundle_adjuster.cc"
#undef private
#undef protected
#include "../ba_step_api.h"

using namespace pano;

namespace {

std::vector<Camera> make_cameras(int n_cam, const double* cams) {
  std::vector<Camera> cs(n_cam);
  for (int i = 0; i < n_cam; ++i) {
    const double* c = cams + 12 * i;
    cs[i].focal = c[0]; cs[i].ppx = c[1]; cs[i].ppy = c[2]; cs[i].aspect = 1;
    for (int k = 0; k < 9; ++k) cs[i].R.data[k] = c[3 + k];
  }
  return cs;
}

// what optimize() does before the first calcError / get_param_update (:118-129); every camera must appear
// in a pair so that slots are camera indices
bool setup(IncrementalBundleAdjuster& ba, std::vector<MatchInfo>& infos, const std::vector<Camera>& cameras, int n_pair,
           const orc_ba_pair* pairs, const double* pts, IncrementalBundleAdjuster::ParamState& state) {
  for (int p = 0; p < n_pair; ++p) {
    for (int k = 0; k < pairs[p].n_match; ++k) {
      const double* q = pts + 4 * (size_t)(pairs[p].match_begin + k);
      infos[p].match.emplace_back(Vec2D(q[0], q[1]), Vec2D(q[2], q[3]));
    }
    ba.add_match(pairs[p].from, pairs[p].to, infos[p]);
  }
  ba.update_index_map();
  if (ba.idx_added.size() != cameras.size()) return false;
  const int nr_img = (int)ba.idx_added.size();
  ba.J = Eigen::MatrixXd{2 * ba.nr_pointwise_match, 6 * nr_img};
  ba.JtJ = Eigen::MatrixXd{6 * nr_img, 6 * nr_img};
  for (auto& idx : ba.idx_added) state.cameras.emplace_back(cameras[idx]);
  return true;
}

}  // namespace

extern "C" int ref_ba_error(int n_cam, const double* cams, int n_pair, const orc_ba_pair* pairs, const double* pts,
                            double* residuals, double* avg, double* max, double* hto) {
  std::vector<Camera> cameras = make_cameras(n_cam, cams);
  IncrementalBundleAdjuster ba(cameras);
  std::vector<MatchInfo> infos(n_pair);                 // MatchPair keeps a reference (incremental_bundle_adjuster.hh:55-60)
  IncrementalBundleAdjuster::ParamState state;
  if (!setup(ba, infos, cameras, n_pair, pairs, pts, state)) return -1;
  auto st = ba.calcError(state);
  for (size_t i = 0; i < st.residuals.size(); ++i) residuals[i] = st.residuals[i];
  *avg = st.avg;
  *max = st.max;
  for (int p = 0; p < n_pair; ++p) {                    // :181-183, the same operations on the same cameras
    const Camera &c_from = state.cameras[ba.index_map[pairs[p].from]], &c_to = state.cameras[ba.index_map[pairs[p].to]];
    Homography h = (c_from.K() * c_from.R) * (c_to.Rinv() * c_to.K().inverse());
    for (int k = 0; k < 9; ++k) hto[9 * p + k] = h.data[k];
  }
  return 0;
}

extern "C" int ref_ba_jtr(int n_cam, const double* cams, int n_pair, const orc_ba_pair* pairs, const double* pts,
                          const double* residuals, double* b) {
  std::vector<Camera> cameras = make_cameras(n_cam, cams);
  IncrementalBundleAdjuster ba(cameras);
  std::vector<MatchInfo> infos(n_pair);
  IncrementalBundleAdjuster::ParamState state;
  if (!setup(ba, infos, cameras, n_pair, pairs, pts, state)) return -1;
  ba.calcJacobianSymbolic(state);                       // get_param_update, :233
  Eigen::Map<const Eigen::VectorXd> err_vec(residuals, 2 * ba.nr_pointwise_match);   // :237
  auto out = ba.J.transpose() * err_vec;                                             // :238
  for (int i = 0; i < out.size(); ++i) b[i] = out(i);
  return 0;
}
