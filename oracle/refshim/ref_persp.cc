// ref_persp.cc — the reference's own CylinderStitcher::perspective_correction (stitch/cylstitcher.cc:139-180)
// behind the checker API of oracle/persp_api.h.  TEST INFRASTRUCTURE ONLY.  Like ref_planet.cc, the reference TUs
// are compiled WHERE THEY LIE by including them (nothing is copied): cylstitcher.cc with the stitcher TUs it needs
// to link.  perspective_correction is protected, so a test subclass of CylinderStitcher sets the `bundle` it reads
// and calls it.  Its getPerspectiveTransform is renamed by macro to a hand-over of the caller's matrix: the
// correction homography is a host solve the engine takes as an input, and the checker build's Eigen stand-in has no
// SVD.  Built by oracle/cyl_sweep.mk with hidden visibility and --gc-sections.
#include <cstring>
#include <string>
#include <vector>
#define getPerspectiveTransform ref_persp_handed_transform
#include "stitch/cylstitcher.cc"
#include "stitch/stitcherbase.cc"
#include "stitch/stitcher_image.cc"
#undef getPerspectiveTransform
#include "../persp_api.h"

namespace pano {
namespace {
const double* g_inv = nullptr;
std::vector<Vec2D> g_p1, g_p2;   // the points perspective_correction handed to getPerspectiveTransform

// The bundle perspective_correction reads: three images (first, identity, last) of the given (warped) shapes, the
// first and last components' homo, proj_range.min, and the flat projection CylinderStitcher::build sets.
class PerspProbe : public CylinderStitcher {
 public:
  PerspProbe(const int shapes[6], const double* first_homo, const double* last_homo, double min_x, double min_y)
      : CylinderStitcher(std::vector<std::string>{"<first>", "<identity>", "<last>"}) {
    for (int k = 0; k < 3; ++k) { imgs[k]._width = shapes[2 * k]; imgs[k]._height = shapes[2 * k + 1]; }
    bundle.identity_idx = 1;
    bundle.proj_method = ConnectedImages::ProjectionMethod::flat;
    bundle.proj_range.min = Vec2D(min_x, min_y);
    double a[9], b[9];
    memcpy(a, first_homo, sizeof(a));
    memcpy(b, last_homo, sizeof(b));
    bundle.component.front().homo = Homography(a);
    bundle.component.back().homo = Homography(b);
  }
  Mat32f correct(const Mat32f& m) { return perspective_correction(m); }
};
}  // namespace

Matrix ref_persp_handed_transform(const std::vector<Vec2D>& p1, const std::vector<Vec2D>& p2) {
  g_p1 = p1;
  g_p2 = p2;
  Matrix m(3, 3);
  memcpy(m.ptr(), g_inv, 9 * sizeof(double));
  return m;
}
}  // namespace pano

extern "C" __attribute__((visibility("default"))) int ref_persp_correction(const float* mosaic, int w, int h,
                                                                           const double inv[9], int lazy_read,
                                                                           int ordered_input, float* out) {
  if (!mosaic || !inv || !out || w < 1 || h < 1) return -1;
  config::LAZY_READ = lazy_read != 0;
  config::ORDERED_INPUT = ordered_input != 0;
  pano::g_inv = inv;
  Mat32f m(h, w, 3);
  memcpy(m.ptr(), mosaic, sizeof(float) * 3 * (size_t)w * h);
  const int shapes[6] = {100, 100, 100, 100, 100, 100};
  const double eye[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  pano::PerspProbe probe(shapes, eye, eye, 0, 0);   // the corners go to the hand-over, which ignores them
  Mat32f res = probe.correct(m);
  if (res.width() != w || res.height() != h) return -1;
  memcpy(out, res.ptr(), sizeof(float) * 3 * (size_t)w * h);
  return 0;
}

extern "C" __attribute__((visibility("default"))) int ref_persp_points(const int shapes[6], const double first_homo[9],
                                                                       const double last_homo[9], double proj_min_x,
                                                                       double proj_min_y, int w, int h,
                                                                       double corners[8], double targets[8]) {
  if (!shapes || !first_homo || !last_homo || !corners || !targets || w < 1 || h < 1) return -1;
  const double eye[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  pano::g_inv = eye;
  pano::g_p1.clear();
  pano::g_p2.clear();
  Mat32f m(h, w, 3);
  memset(m.ptr(), 0, sizeof(float) * 3 * (size_t)w * h);
  pano::PerspProbe probe(shapes, first_homo, last_homo, proj_min_x, proj_min_y);
  probe.correct(m);
  if (pano::g_p1.size() != 4 || pano::g_p2.size() != 4) return -1;
  for (int q = 0; q < 4; ++q) {
    corners[2 * q] = pano::g_p1[q].x; corners[2 * q + 1] = pano::g_p1[q].y;
    targets[2 * q] = pano::g_p2[q].x; targets[2 * q + 1] = pano::g_p2[q].y;
  }
  return 0;
}
