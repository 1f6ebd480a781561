// cyl_blend_test.cc — compiles the drop-in's B200CylinderBlender (openpano_b200/host/pano_host.hh) against the
// REFERENCE's headers and runs it next to cylinder mode's own path: CylinderWarper(h_factor).warp of every image
// (stitch/warp.cc), then LinearBlender (LAZY_READ 1 and 0) or MultiBandBlender over the warped images, driven as
// ConnectedImages::blend drives them with the flat projection (stitcher_image.cc:116-155), from
// oracle/_ref/libopenpano_ref.so.  The drop-in gets the UNWARPED images, windows of 1, 2 and all of them; every
// output float must be bit-identical, and every ImageRef must be released by run().
// Built by oracle/cyl_blend.mk (needs the reference sources); run by tests/test_gpu_blend_cyl.py on a GPU.
//   cyl_blend_test <stack.bin>   stack.bin: int32 n, w, h, then n*h*w*3 float32 (unwarped), then float64
//                                h_factor, then per image int32 x0,y0,x1,y1 + float64 homo_inv[9] of the WARPED
//                                image, then float64 res, min_x, min_y
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#include "pano_host.hh"
#include "stitch/multiband.hh"
#include "stitch/projection.hh"
#include "stitch/warp.hh"

using namespace pano;
using namespace pano_b200;

static int g_fail = 0;
#define CHECK(cond, ...) do { if (!(cond)) { ++g_fail; printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } while (0)

struct Item { int x0, y0, x1, y1; double hi[9]; };

// ImageRefs with the images attached, as after ImageRef::load (load() is a no-op while a Mat is attached)
static std::vector<std::unique_ptr<ImageRef>> attach(const std::vector<Mat32f>& imgs) {
  std::vector<std::unique_ptr<ImageRef>> refs;
  for (auto& m : imgs) {
    refs.emplace_back(new ImageRef("<memory>"));
    refs.back()->img = new Mat32f(m.clone());
    refs.back()->_width = m.width(); refs.back()->_height = m.height();
  }
  return refs;
}

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: cyl_blend_test stack.bin\n"); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  int hdr[3];
  if (fread(hdr, 4, 3, f) != 3) return 2;
  const int n = hdr[0], w = hdr[1], h = hdr[2];
  std::vector<Mat32f> imgs;
  for (int k = 0; k < n; ++k) {
    Mat32f m(h, w, 3);
    if (fread(m.ptr(), sizeof(float), (size_t)w * h * 3, f) != (size_t)w * h * 3) return 2;
    imgs.push_back(m);
  }
  double h_factor;
  if (fread(&h_factor, 8, 1, f) != 1) return 2;
  std::vector<Item> items(n);
  for (int k = 0; k < n; ++k) {
    if (fread(&items[k].x0, 4, 4, f) != 4) return 2;
    if (fread(items[k].hi, 8, 9, f) != 9) return 2;
  }
  double geo[3];
  if (fread(geo, 8, 3, f) != 3) return 2;
  fclose(f);
  config::FOCAL_LENGTH = 37;           // config.cfg's values: the warp's radius and the multiband blur windows
  config::GAUSS_WINDOW_FACTOR = 6;

  // cylstitcher.cc:65-67: the reference's own warp of every image (its keypoints play no part in the blend)
  std::vector<Mat32f> warped;
  {
    CylinderWarper warper(h_factor);
    for (auto& m : imgs) {
      Mat32f x = m.clone();
      std::vector<Vec2D> kpts;
      warper.warp(x, kpts);
      warped.push_back(x);
    }
  }

  Context ctx(0);
  Vec2D resolution(geo[0], geo[0]), proj_min(geo[1], geo[2]);
  const int cases[5][3] = {{0, 1, 1}, {0, 0, 1}, {0, 1, 0}, {2, 1, 1}, {5, 1, 1}};   // (bands, LAZY_READ, ORDERED_INPUT)
  for (auto& cs : cases) {
    const int bands = cs[0];
    config::LAZY_READ = cs[1] != 0;
    config::ORDERED_INPUT = cs[2] != 0;
    config::MULTIBAND = bands;
    Mat32f want;
    {
      auto refs = attach(warped);
      std::unique_ptr<BlenderBase> rb;
      if (bands > 0) rb.reset(new MultiBandBlender{bands}); else rb.reset(new LinearBlender);
      for (int k = 0; k < n; ++k) {
        Homography homo_inv(items[k].hi);
        Shape2D shp{warped[k].width(), warped[k].height()};
        rb->add_image(Coor(items[k].x0, items[k].y0), Coor(items[k].x1, items[k].y1), *refs[k],
                      [=](Coor t) -> Vec2D {                           // stitcher_image.cc:142-151
                        Vec2D c = Vec2D(t.x, t.y) * resolution + proj_min;
                        Vec ret = homo_inv.trans(flat::proj2homo(Vec2D(c.x, c.y)));
                        if (ret.z < 0) return Vec2D{-10, -10};
                        double denom = 1.0 / ret.z;
                        return Vec2D{ret.x * denom, ret.y * denom} + shp.center();
                      });
      }
      want = rb->run();
    }
    for (int window : {1, 2, n}) {
      auto refs = attach(imgs);
      B200CylinderBlender mine(ctx, bands, h_factor, resolution, proj_min, window);
      for (int k = 0; k < n; ++k)
        mine.add_image(Coor(items[k].x0, items[k].y0), Coor(items[k].x1, items[k].y1), *refs[k], Homography(items[k].hi));
      Mat32f got = mine.run();
      int loaded = 0;
      for (auto& r : refs) loaded += r->img != nullptr;
      CHECK(loaded == 0, "bands=%d lazy=%d ordered=%d window=%d: %d images still loaded after run()", bands, cs[1], cs[2],
            window, loaded);
      const bool same = got.width() == want.width() && got.height() == want.height() &&
                        memcmp(got.ptr(), want.ptr(), sizeof(float) * (size_t)got.width() * got.height() * 3) == 0;
      CHECK(same, "bands=%d lazy=%d ordered=%d window=%d: mosaic differs", bands, cs[1], cs[2], window);
      if (same)
        printf("bands=%d lazy=%d ordered=%d window=%d: %dx%d identical\n", bands, cs[1], cs[2], window, got.width(),
               got.height());
    }
  }
  printf(g_fail ? "CYL BLEND TEST FAILED (%d)\n" : "CYL BLEND TEST OK\n", g_fail);
  return g_fail ? 1 : 0;
}
