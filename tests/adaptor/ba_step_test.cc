// ba_step_test.cc — compiles the drop-in's bundle-adjustment step (B200BundleAdjusterStep,
// openpano_b200/host/pano_host.hh) against the REFERENCE's headers and runs it next to the reference's
// own IncrementalBundleAdjuster members (stitch/incremental_bundle_adjuster.cc, from
// oracle/_ref/libopenpano_ref.so):
//   error(cameras)         vs calcError(state)                                   (:171-220)
//   normal_equations(...)  vs calcJacobianSymbolic(state) + J.transpose() * err_vec  (:233-238)
// and the LM sequence error(state) -> normal_equations -> error(rejected state) -> normal_equations,
// whose second b must use the rejected state's residuals with the kept state's J (:140, :152-153).
// Everything must be bit-identical.  A whole optimize() is not run: the checker build's Eigen stand-in
// has no solver (colPivHouseholderQr().solve() aborts), so the damping and the solve are not exercised.
// Built by oracle/ba_step.mk (needs the reference sources); run by tests/test_gpu_ba_step.py on a GPU.
//   ba_step_test <case.bin>   case.bin: int32 n_cam, n_pair; n_pair x int32 {from, to, n_match};
//                             float64 cams[n_cam][12], rejected[n_cam][12] ({focal, ppx, ppy, R[9]});
//                             float64 pts[n_match][4] (to.x, to.y, from.x, from.y)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <set>
#include <limits>

#include "pano_host.hh"
#include "../../oracle/oracle_api.h"
#define private public            // calcError, calcJacobianSymbolic, J, JtJ, index_map ... are private members
#define protected public
#include "stitch/incremental_bundle_adjuster.hh"
#undef private
#undef protected

using namespace pano;
using namespace pano_b200;

static int g_fail = 0;
#define CHECK(cond, ...) do { if (!(cond)) { ++g_fail; printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } while (0)

static bool same(const double* a, const double* b, size_t n) { return n == 0 || memcmp(a, b, n * sizeof(double)) == 0; }

static std::vector<Camera> make_cameras(int n, const double* c) {
  std::vector<Camera> cs(n);
  for (int i = 0; i < n; ++i) {
    cs[i].focal = c[12 * i]; cs[i].ppx = c[12 * i + 1]; cs[i].ppy = c[12 * i + 2]; cs[i].aspect = 1;
    for (int k = 0; k < 9; ++k) cs[i].R.data[k] = c[12 * i + 3 + k];
  }
  return cs;
}

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: ba_step_test case.bin\n"); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  int hdr[2];
  if (fread(hdr, 4, 2, f) != 2) return 2;
  const int n_cam = hdr[0], n_pair = hdr[1];
  std::vector<orc_ba_pair> pairs(n_pair);
  int nm = 0;
  for (int p = 0; p < n_pair; ++p) {
    int v[3];
    if (fread(v, 4, 3, f) != 3) return 2;
    memset(&pairs[p], 0, sizeof(orc_ba_pair));
    pairs[p].from = v[0]; pairs[p].to = v[1]; pairs[p].match_begin = nm; pairs[p].n_match = v[2];
    nm += v[2];
  }
  std::vector<double> cams(12 * n_cam), rejected(12 * n_cam), pts(4 * (size_t)nm);
  if (fread(cams.data(), 8, cams.size(), f) != cams.size() || fread(rejected.data(), 8, rejected.size(), f) != rejected.size() ||
      fread(pts.data(), 8, pts.size(), f) != pts.size()) return 2;
  fclose(f);

  // the reference's adjuster, set up as optimize() sets it up (:118-129)
  std::vector<Camera> cameras = make_cameras(n_cam, cams.data());
  IncrementalBundleAdjuster ba(cameras);
  std::vector<MatchInfo> infos(n_pair);
  for (int p = 0; p < n_pair; ++p) {
    for (int k = 0; k < pairs[p].n_match; ++k) {
      const double* q = &pts[4 * (size_t)(pairs[p].match_begin + k)];
      infos[p].match.emplace_back(Vec2D(q[0], q[1]), Vec2D(q[2], q[3]));
    }
    ba.add_match(pairs[p].from, pairs[p].to, infos[p]);
  }
  ba.update_index_map();
  const int nr_img = (int)ba.idx_added.size();
  if (nr_img != n_cam) { printf("every camera must appear in a pair\n"); return 2; }
  ba.J = Eigen::MatrixXd{2 * ba.nr_pointwise_match, 6 * nr_img};
  ba.JtJ = Eigen::MatrixXd{6 * nr_img, 6 * nr_img};
  IncrementalBundleAdjuster::ParamState state, new_state;
  for (auto& idx : ba.idx_added) state.cameras.emplace_back(cameras[idx]);
  std::vector<Camera> rej = make_cameras(n_cam, rejected.data());
  for (auto& idx : ba.idx_added) new_state.cameras.emplace_back(rej[idx]);

  Context ctx(0);
  std::vector<B200BundleAdjusterStep::Pair> sp;
  for (size_t p = 0; p < ba.match_pairs.size(); ++p)
    sp.push_back({ba.index_map[ba.match_pairs[p].from], ba.index_map[ba.match_pairs[p].to], &ba.match_pairs[p].m});
  B200BundleAdjusterStep step(ctx, nr_img, sp);

  // ---- calcError
  auto want = ba.calcError(state);
  std::vector<double> res;
  auto got = step.error(state.cameras, &res);
  CHECK(res.size() == want.residuals.size() && same(res.data(), want.residuals.data(), res.size()), "residuals differ");
  CHECK(same(&got.avg, &want.avg, 1), "avg %.17g vs %.17g", got.avg, want.avg);
  CHECK(same(&got.max, &want.max, 1), "max %.17g vs %.17g", got.max, want.max);
  printf("calcError: %zu residuals, avg %.6f, max %.6f\n", res.size(), got.avg, got.max);

  // ---- get_param_update up to the damping, at `state`
  std::vector<double> mats(117 * (size_t)n_pair + 1);
  {
    std::vector<orc_ba_pair> tmp = pairs;                  // the 13 matrices by the reference's own operations
    if (ref_ba_pair_mats(n_cam, cams.data(), n_pair, tmp.data()) != 0) return 2;
    for (int p = 0; p < n_pair; ++p) memcpy(&mats[117 * (size_t)p], tmp[p].m, sizeof(tmp[p].m));
  }
  const int N = 6 * nr_img;
  auto jacobian_and_b = [&](const std::vector<double>& residuals, const char* what) {
    ba.calcJacobianSymbolic(state);
    Eigen::Map<const Eigen::VectorXd> err_vec(residuals.data(), 2 * ba.nr_pointwise_match);
    Eigen::VectorXd b_want = ba.J.transpose() * err_vec;
    std::vector<double> jtj, b, rows;
    step.normal_equations(mats, jtj, b, &rows);
    CHECK(same(jtj.data(), ba.JtJ.d.data(), (size_t)N * N), "%s: JtJ differs", what);
    CHECK(same(b.data(), b_want.d.data(), (size_t)N), "%s: b differs", what);
    bool rows_ok = true;
    for (int p = 0; p < n_pair && rows_ok; ++p) {
      const int pf = ba.index_map[pairs[p].from] * 6, pt = ba.index_map[pairs[p].to] * 6;
      for (int k = 0; k < pairs[p].n_match && rows_ok; ++k) {
        const int m = pairs[p].match_begin + k;
        const double* r = &rows[24 * (size_t)m];
        for (int i = 0; i < 6; ++i)
          rows_ok = rows_ok && same(&r[i], &ba.J(2 * m, pf + i), 1) && same(&r[6 + i], &ba.J(2 * m, pt + i), 1) &&
                    same(&r[12 + i], &ba.J(2 * m + 1, pf + i), 1) && same(&r[18 + i], &ba.J(2 * m + 1, pt + i), 1);
      }
    }
    CHECK(rows_ok, "%s: J rows differ", what);
    printf("%s: J %d x %d, JtJ %d x %d, b[0] %.6g ok\n", what, 2 * nm, N, N, N, b.empty() ? 0.0 : b[0]);
  };
  jacobian_and_b(want.residuals, "get_param_update(state)");

  // ---- a rejected step: calcError(new_state) (:146), then the next get_param_update still at `state` (:140)
  auto want2 = ba.calcError(new_state);
  auto got2 = step.error(new_state.cameras);
  CHECK(same(&got2.avg, &want2.avg, 1) && same(&got2.max, &want2.max, 1), "rejected state: avg/max differ");
  jacobian_and_b(want2.residuals, "get_param_update after a rejected step");

  printf(g_fail ? "BA STEP TEST FAILED (%d)\n" : "BA STEP TEST OK\n", g_fail);
  return g_fail ? 1 : 0;
}
