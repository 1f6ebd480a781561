// lazy_sift_test.cc — compiles the drop-in's B200SIFTDetector::detect_lazy (openpano_b200/host/pano_host.hh) against
// the REFERENCE's headers and runs it next to the reference's calc_feature loop (stitcherbase.cc:14-19): ImageRef::load
// (read_img, CImg's PNM reader) + SIFTDetector::detect_feature, both from oracle/_ref/libopenpano_ref.so.
// The program writes PPM (3 channels) and PGM (grey) files of synthetic pixels of several shapes and detects them
// through ImageRefs at several window sizes.  Coordinates and descriptors must be bit-identical, and every image must
// be released afterwards, as LAZY_READ leaves them.
// Built by oracle/lazy_sift.mk (needs the reference sources); run by tests/test_gpu_sift_stream.py on a GPU.
//   lazy_sift_test <dir>     dir: where the image files are written
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "pano_host.hh"
#include "lib/imgproc.hh"
#include "stitch/imageref.hh"

using namespace pano;
using namespace pano_b200;

static int g_fail = 0;
#define CHECK(cond, ...) do { if (!(cond)) { ++g_fail; printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } while (0)

static void set_config(const pano_params& p) {   // what init_config() does from config.cfg (main.cc:237-292)
  using namespace config;
  CYLINDER = false; TRANS = false; CROP = true; ESTIMATE_CAMERA = true; STRAIGHTEN = true;
  FOCAL_LENGTH = p.focal_length; MAX_OUTPUT_SIZE = p.max_output_size; ORDERED_INPUT = p.ordered_input != 0;
  LAZY_READ = p.lazy_read != 0; SIFT_WORKING_SIZE = p.sift_working_size; NUM_OCTAVE = p.num_octave;
  NUM_SCALE = p.num_scale; SCALE_FACTOR = p.scale_factor; GAUSS_SIGMA = p.gauss_sigma;
  GAUSS_WINDOW_FACTOR = p.gauss_window_factor; JUDGE_EXTREMA_DIFF_THRES = p.judge_extrema_diff_thres;
  CONTRAST_THRES = p.contrast_thres; PRE_COLOR_THRES = p.pre_color_thres; EDGE_RATIO = p.edge_ratio;
  CALC_OFFSET_DEPTH = p.calc_offset_depth; OFFSET_THRES = p.offset_thres; ORI_RADIUS = p.ori_radius;
  ORI_HIST_SMOOTH_COUNT = p.ori_hist_smooth_count; DESC_HIST_SCALE_FACTOR = p.desc_hist_scale_factor;
  DESC_INT_FACTOR = p.desc_int_factor; MATCH_REJECT_NEXT_RATIO = p.match_reject_next_ratio;
  MULTIBAND = p.multiband;
}

static bool same_desc(const std::vector<Descriptor>& a, const std::vector<Descriptor>& b) {
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); ++i) {
    if (memcmp(&a[i].coor, &b[i].coor, sizeof(Vec2D)) != 0) return false;
    if (a[i].descriptor.size() != b[i].descriptor.size()) return false;
    if (memcmp(a[i].descriptor.data(), b[i].descriptor.data(), a[i].descriptor.size() * sizeof(float)) != 0) return false;
  }
  return true;
}

// Discs of random colour over a smooth gradient plus a little noise: blob and corner features at every scale.
static std::vector<unsigned char> synth(int w, int h, int ch, unsigned seed) {
  unsigned s = seed * 2654435761u + 12345u;
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (s >> 8) & 0xffffff; };
  std::vector<float> img((size_t)w * h * ch);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < ch; ++c) img[((size_t)y * w + x) * ch + c] = 60.f + 80.f * (float)(x + (c + 1) * y) / (float)(w + 3 * h);
  const int discs = (w * h) / 2500;
  for (int d = 0; d < discs; ++d) {
    const int cx = rnd() % w, cy = rnd() % h, r = 3 + rnd() % 24;
    float col[3];
    for (int c = 0; c < 3; ++c) col[c] = (float)(rnd() % 256);
    for (int y = std::max(0, cy - r); y < std::min(h, cy + r + 1); ++y)
      for (int x = std::max(0, cx - r); x < std::min(w, cx + r + 1); ++x)
        if ((x - cx) * (x - cx) + (y - cy) * (y - cy) <= r * r)
          for (int c = 0; c < ch; ++c) img[((size_t)y * w + x) * ch + c] = col[c];
  }
  std::vector<unsigned char> pix(img.size());
  for (size_t i = 0; i < img.size(); ++i) {
    const float v = img[i] + (float)((int)(rnd() % 9) - 4);
    pix[i] = (unsigned char)std::min(255.f, std::max(0.f, v));
  }
  return pix;
}

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: lazy_sift_test <dir>\n"); return 2; }
  pano_params p;
  pano_params_default(&p);
  set_config(p);
  Context ctx(0);
  SIFTDetector ref_det;
  B200SIFTDetector det(ctx);

  struct Case { int w, h, ch; };
  const Case cases[] = {{640, 480, 3}, {500, 375, 1}, {333, 517, 3}, {640, 480, 3}, {1300, 867, 1}, {640, 480, 3}, {401, 299, 3}};
  const int n = sizeof(cases) / sizeof(cases[0]);
  std::vector<std::string> paths(n);
  for (int k = 0; k < n; ++k) {
    const Case& c = cases[k];
    const std::vector<unsigned char> pix = synth(c.w, c.h, c.ch, 29 + k);
    paths[k] = std::string(argv[1]) + "/img" + std::to_string(k) + (c.ch == 3 ? ".ppm" : ".pgm");
    FILE* f = fopen(paths[k].c_str(), "wb");
    if (!f) { perror(paths[k].c_str()); return 2; }
    fprintf(f, "%s\n%d %d\n255\n", c.ch == 3 ? "P6" : "P5", c.w, c.h);
    fwrite(pix.data(), 1, pix.size(), f);
    fclose(f);
  }

  // the reference: calc_feature's loop body with LAZY_READ 1
  std::vector<std::vector<Descriptor>> want(n);
  {
    std::vector<ImageRef> imgs;
    imgs.reserve(n);
    for (int k = 0; k < n; ++k) imgs.emplace_back(paths[k]);
    for (int k = 0; k < n; ++k) {
      imgs[k].load();
      want[k] = ref_det.detect_feature(*imgs[k].img);
      imgs[k].release();
      CHECK(!want[k].empty(), "image %d: no reference features", k);
    }
  }

  for (int window : {1, 3, n}) {
    std::vector<ImageRef> imgs;
    imgs.reserve(n);
    for (int k = 0; k < n; ++k) imgs.emplace_back(paths[k]);
    if (window == 3) imgs[2].load();   // an image already resident when detection starts
    auto got = det.detect_lazy(imgs, window);
    CHECK((int)got.size() == n, "window %d: %zu feature lists for %d images", window, got.size(), n);
    for (int k = 0; k < n && k < (int)got.size(); ++k) {
      const bool same = same_desc(want[k], got[k]);
      CHECK(same, "window %d, image %d (%dx%d, %d channels): %zu reference descriptors, %zu from detect_lazy", window, k,
            cases[k].w, cases[k].h, cases[k].ch, want[k].size(), got[k].size());
      CHECK(imgs[k].img == nullptr, "window %d, image %d still loaded", window, k);
      CHECK(imgs[k].width() == cases[k].w && imgs[k].height() == cases[k].h, "window %d, image %d: shape %dx%d", window, k,
            imgs[k].width(), imgs[k].height());
      if (same) printf("window %d, image %d (%dx%d, %d channels): %zu descriptors identical\n", window, k, cases[k].w,
                       cases[k].h, cases[k].ch, got[k].size());
    }
  }
  printf(g_fail ? "LAZY SIFT TEST FAILED (%d)\n" : "LAZY SIFT TEST OK\n", g_fail);
  return g_fail ? 1 : 0;
}
