// ref_planet.cc — the reference's own planet() (main.cc:294-331) behind the checker API of
// oracle/planet_api.h.  TEST INFRASTRUCTURE ONLY.  Like ref_ba_step.cc, the reference TU is compiled
// WHERE IT LIES by including it (nothing is copied).  Its file I/O is renamed by macro to an in-memory
// hand-over: read_img returns the caller's image, write_rgb copies planet()'s result out.  main() is
// renamed too.  Built into its own library by oracle/planet.mk with hidden visibility and
// -ffunction-sections / --gc-sections, so that work() and the test_*() drawers, with the Stitcher /
// Eigen code they reference, are dropped by the linker; only planet() and what it calls remain.
#include <memory>
#include <cstring>
#define read_img ref_planet_read_img
#define write_rgb ref_planet_write_rgb
#define main ref_planet_main_unused
#include "main.cc"
#undef main
#undef read_img
#undef write_rgb
#include "../planet_api.h"

namespace pano {
namespace {
const float* g_in = nullptr;
int g_w = 0, g_h = 0;
float* g_out = nullptr;
}  // namespace

Mat32f ref_planet_read_img(const char*) {
  Mat32f m(g_h, g_w, 3);
  memcpy(m.ptr(), g_in, sizeof(float) * 3 * (size_t)g_w * g_h);
  return m;
}

void ref_planet_write_rgb(const char*, const Mat32f& m) {
  memcpy(g_out, m.ptr(), sizeof(float) * 3 * (size_t)m.width() * m.height());
}
}  // namespace pano

extern "C" __attribute__((visibility("default"))) int ref_planet(const float* rgb_hwc, int w, int h, float* out_hwc) {
  if (w < 1 || h < 1) return -1;
  pano::g_in = rgb_hwc; pano::g_w = w; pano::g_h = h; pano::g_out = out_hwc;
  planet("in-memory");
  return 0;
}
