// cyl_sweep_test.cc — compiles B200CylinderBlender::write_sweep (openpano_b200/host/pano_host_io.hh) against the
// REFERENCE's headers and runs it next to cylinder mode's own output end: read_img of each file,
// CylinderWarper(h_factor).warp, LinearBlender (LAZY_READ 1 and 0) or MultiBandBlender{5} driven as
// ConnectedImages::blend drives them with the flat projection (oracle/_ref/libopenpano_ref.so), then
// CylinderStitcher::perspective_correction (oracle/_ref/libopenpano_ref_persp.so, its homography handed over), crop()
// and write_rgb() to a .png and a .ppm — against write_sweep of the same files, file bytes.  6 views of 200×150, PNG
// (RGBA) and PPM sources mixed; a mild and a strongly keystoned correction; strips of 1, 21 and 400 rows (one strip
// of the whole canvas); keep budgets of 0 and no limit.  Each run must load an image exactly once per upload.
// The corner points write_sweep(bundle, ...) solves perspective_correction's homography from
// (b200_correction_points) must be the ones the reference's perspective_correction hands to getPerspectiveTransform,
// bit for bit, for random bundles (ref_persp_points).
// Built by oracle/cyl_sweep.mk (needs the reference sources); run by tests/test_gpu_cyl_sweep.py on a GPU.
//   cyl_sweep_test <dir>     dir: where the image files are written
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "pano_host.hh"
#include "pano_host_io.hh"
#include "lib/imgproc.hh"
#include "stitch/multiband.hh"
#include "stitch/projection.hh"
#include "stitch/warp.hh"
#include "stitch/stitcher_image.hh"
#include "persp_api.h"

using namespace pano;
using namespace pano_b200;

static int g_fail = 0;
#define CHECK(cond, ...) do { if (!(cond)) { ++g_fail; printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } while (0)

static std::vector<unsigned char> file_bytes(const std::string& path) {
  std::vector<unsigned char> out;
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return out;
  unsigned char buf[65536];
  size_t n;
  while ((n = fread(buf, 1, sizeof buf, f)) > 0) out.insert(out.end(), buf, buf + n);
  fclose(f);
  return out;
}

static unsigned g_seed = 4242u;
static unsigned rnd() { g_seed = g_seed * 1664525u + 1013904223u; return (g_seed >> 8) & 0xffffff; }

// w×h×3 pixels: a gradient with random discs and a little noise
static std::vector<unsigned char> synth_rgb(int w, int h) {
  std::vector<unsigned char> pix((size_t)w * h * 3);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < 3; ++c)
        pix[((size_t)y * w + x) * 3 + c] = (unsigned char)(40 + (150 * (x + (c + 1) * y)) / (w + 3 * h) + rnd() % 7);
  for (int d = 0; d < (w * h) / 1500; ++d) {
    const int cx = rnd() % w, cy = rnd() % h, r = 3 + rnd() % 15;
    unsigned char col[3] = {(unsigned char)(rnd() & 255), (unsigned char)(rnd() & 255), (unsigned char)(rnd() & 255)};
    for (int y = std::max(0, cy - r); y < std::min(h, cy + r + 1); ++y)
      for (int x = std::max(0, cx - r); x < std::min(w, cx + r + 1); ++x)
        if ((x - cx) * (x - cx) + (y - cy) * (y - cy) <= r * r)
          for (int c = 0; c < 3; ++c) pix[((size_t)y * w + x) * 3 + c] = col[c];
  }
  return pix;
}

// an RGBA PNG (random alpha, which read_img ignores) or a PPM of the pixels
static bool write_file(const std::string& path, const std::vector<unsigned char>& rgb, int w, int h) {
  if (endswith(path.c_str(), ".png")) {
    std::vector<unsigned char> rgba((size_t)w * h * 4);
    for (size_t i = 0; i < (size_t)w * h; ++i) {
      memcpy(&rgba[i * 4], &rgb[i * 3], 3);
      rgba[i * 4 + 3] = (unsigned char)(rnd() & 255);
    }
    return lodepng::encode(path, rgba, (unsigned)w, (unsigned)h) == 0;
  }
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) return false;
  fprintf(f, "P6\n%d %d\n255\n", w, h);
  fwrite(rgb.data(), 1, rgb.size(), f);
  fclose(f);
  return true;
}

struct View { std::string path; Coor ul, br; Homography hi; };

// Cylinder mode's output end on read_img's images: warp, blend, perspective_correction with `inv`, crop, write_rgb.
static void reference_write(const std::vector<View>& views, double h_factor, int bands, Vec2D resolution,
                            Vec2D proj_min, const double inv[9], const std::string& out) {
  std::vector<std::unique_ptr<ImageRef>> refs;
  std::unique_ptr<BlenderBase> rb;
  if (bands > 0) rb.reset(new MultiBandBlender{bands}); else rb.reset(new LinearBlender);
  CylinderWarper warper(h_factor);
  for (auto& v : views) {
    Mat32f m = read_img(v.path.c_str());
    std::vector<Vec2D> kpts;
    warper.warp(m, kpts);                                    // cylstitcher.cc:65-67
    refs.emplace_back(new ImageRef("<memory>"));
    refs.back()->img = new Mat32f(m);
    refs.back()->_width = m.width(); refs.back()->_height = m.height();
    const Homography homo_inv = v.hi;
    Shape2D shp{m.width(), m.height()};
    rb->add_image(v.ul, v.br, *refs.back(), [=](Coor t) -> Vec2D {   // stitcher_image.cc:142-151
      Vec2D c = Vec2D(t.x, t.y) * resolution + proj_min;
      Vec ret = homo_inv.trans(flat::proj2homo(Vec2D(c.x, c.y)));
      if (ret.z < 0) return Vec2D{-10, -10};
      double denom = 1.0 / ret.z;
      return Vec2D{ret.x * denom, ret.y * denom} + shp.center();
    });
  }
  Mat32f res = rb->run();
  Mat32f corrected(res.height(), res.width(), 3);
  if (ref_persp_correction(res.ptr(), res.width(), res.height(), inv, config::LAZY_READ, config::ORDERED_INPUT,
                           corrected.ptr()))
    error_exit("ref_persp_correction failed");
  write_rgb(out.c_str(), crop(corrected));
}

// b200_correction_points against the points the reference's perspective_correction computes, on random bundles:
// shapes, projective homographies of the first and last components, proj_range.min and mosaic sizes.
static void compare_points() {
  for (int t = 0; t < 50; ++t) {
    int shapes[6];
    for (int q = 0; q < 6; ++q) shapes[q] = 2 + (int)(rnd() % 3000);
    double hf[9], hl[9];
    for (int q = 0; q < 9; ++q) {
      const double u = (double)(rnd() % 2001) / 1000.0 - 1.0;   // [-1, 1]
      hf[q] = (q % 4 == 0 ? 1.0 : 0.0) + (q >= 6 ? 1e-4 : q == 2 || q == 5 ? 900.0 : 0.1) * u;
      hl[q] = (q % 4 == 0 ? 1.0 : 0.0) + (q >= 6 ? 1e-4 : q == 2 || q == 5 ? 900.0 : 0.1) * (u * 0.7 - 0.2);
    }
    const double mx = -(double)(rnd() % 5000) - 0.25, my = -(double)(rnd() % 3000) - 0.5;
    const int w = 2 + (int)(rnd() % 9000), h = 2 + (int)(rnd() % 3000);
    double want_c[8], want_t[8];
    if (ref_persp_points(shapes, hf, hl, mx, my, w, h, want_c, want_t)) { CHECK(false, "ref_persp_points failed"); continue; }
    std::vector<ImageRef> imgs;
    for (int k = 0; k < 3; ++k) imgs.emplace_back("<memory>");
    ConnectedImages bundle;
    bundle.component.resize(3);
    for (int k = 0; k < 3; ++k) bundle.component[k].imgptr = &imgs[k];
    bundle.identity_idx = 1;
    bundle.proj_method = ConnectedImages::ProjectionMethod::flat;
    bundle.proj_range.min = Vec2D(mx, my);
    bundle.component.front().homo = Homography(hf);
    bundle.component.back().homo = Homography(hl);
    std::vector<Vec2D> corners, targets;
    b200_correction_points(bundle, shapes[2], shapes[3], shapes[0], shapes[1], shapes[4], shapes[5], w, h, &corners,
                           &targets);
    bool same = corners.size() == 4 && targets.size() == 4;
    for (int q = 0; same && q < 4; ++q) {
      const double got[4] = {corners[q].x, corners[q].y, targets[q].x, targets[q].y};
      const double want[4] = {want_c[2 * q], want_c[2 * q + 1], want_t[2 * q], want_t[2 * q + 1]};
      same = memcmp(got, want, sizeof(got)) == 0;
    }
    CHECK(same, "bundle %d: the correction's points differ from the reference's", t);
    if (same) printf("bundle %d: correction points identical\n", t);
  }
}

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: cyl_sweep_test <dir>\n"); return 2; }
  const std::string dir = argv[1];
  config::FOCAL_LENGTH = 37;           // config.cfg's values: the warp's radius and the multiband blur windows
  config::GAUSS_WINDOW_FACTOR = 6;
  config::ORDERED_INPUT = true;
  config::CROP = true;
  compare_points();
  Context ctx(0);
  const int W = 200, H = 150;
  const double h_factor = 1.0;
  pano_params p = snapshot_params();
  int ww = 0, wh = 0;
  double ox, oy;
  ctx.check(pano_cyl_warp_shape(W, H, h_factor, &p, &ww, &wh, &ox, &oy));
  std::vector<View> views;
  for (int k = 0; k < 6; ++k) {
    const std::string path = dir + "/view" + std::to_string(k) + (k % 2 ? ".ppm" : ".png");
    if (!write_file(path, synth_rgb(W, H), W, H)) { printf("FAIL: cannot write %s\n", path.c_str()); return 2; }
    const int x = 55 * k, y = 3 * (k % 3);
    const double hi[9] = {1, 0, -(double)x, 0, 1, -(double)y, 0, 0, 1};
    views.push_back(View{path, Coor(x, y), Coor(x + ww - 1, y + wh - 1), Homography(hi)});
  }
  const int cw = 55 * 5 + ww, ch = 6 + wh;
  // perspective_correction's inv: mild, and strongly keystoned (a strip of corrected rows reads many mosaic rows)
  const double mild[9] = {1.01, 0.02, -1.5, -0.01, 0.99, 1.25, 1e-5, 2e-5, 1.0};
  const double keyst[9] = {1.0, 0.35, -0.2 * cw, 0.0, 1.6, -0.3 * ch, 0.0, 2.5 / ch, 1.0};
  Vec2D resolution(1.0, 1.0), proj_min(-ww / 2.0, -wh / 2.0);
  const int cases[4][2] = {{0, 1}, {0, 0}, {5, 1}, {5, 0}};   // (bands, LAZY_READ)
  for (auto& cs : cases)
    for (int ci = 0; ci < 2; ++ci) {
      const double (&inv)[9] = ci ? keyst : mild;
      const int bands = cs[0];
      config::LAZY_READ = cs[1] != 0;
      config::MULTIBAND = bands;
      const char* iname = ci ? "keystone" : "mild";
      for (const char* ext : {".png", ".ppm"}) {
        const std::string ref_path = dir + "/ref_out" + ext;
        reference_write(views, h_factor, bands, resolution, proj_min, inv, ref_path);
        const std::vector<unsigned char> want = file_bytes(ref_path);
        for (size_t keep : {(size_t)0, SIZE_MAX})
          for (int rows : {1, 21, 400}) {
            std::vector<std::unique_ptr<ImageRef>> refs;
            B200CylinderBlender mine(ctx, bands, h_factor, resolution, proj_min);
            for (const View& v : views) {
              refs.emplace_back(new ImageRef(v.path));
              refs.back()->load();                           // the shape, as calc_feature() leaves it
              refs.back()->release();
              mine.add_image(v.ul, v.br, *refs.back(), v.hi);
            }
            const std::string path = dir + "/b200_out" + ext;
            mine.write_sweep(Homography(inv), rows, keep, true, path.c_str());
            const std::vector<unsigned char> got = file_bytes(path);
            const bool same = !want.empty() && want == got;
            const bool once = mine.last_sweep_loads() == mine.last_sweep_uploads();
            CHECK(same && once, "bands=%d lazy=%d %s %s keep=%zu rows=%d: %zu reference bytes, %zu from write_sweep; "
                  "%ld loads for %lld uploads", bands, cs[1], iname, ext, keep, rows, want.size(), got.size(),
                  mine.last_sweep_loads(), mine.last_sweep_uploads());
            if (same && once)
              printf("bands=%d lazy=%d %s %s keep=%zu rows=%d: %zu file bytes identical\n", bands, cs[1], iname, ext,
                     keep, rows, got.size());
          }
      }
    }
  printf(g_fail ? "CYL SWEEP TEST FAILED (%d)\n" : "CYL SWEEP TEST OK\n", g_fail);
  return g_fail ? 1 : 0;
}
