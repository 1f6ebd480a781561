// blend_sweep_test.cc — compiles B200PixelBlender::write_sweep (openpano_b200/host/pano_host_io.hh) against the
// REFERENCE's headers and runs it next to the reference's own work() tail (oracle/_ref/libopenpano_ref.so):
// read_img of each file, LinearBlender (LAZY_READ 1) or MultiBandBlender{5}, crop() and write_rgb() to a .png and a
// .ppm, against write_sweep of the same files (decoded on demand), file bytes.  9 views of 360×270 on a flat
// canvas, PNG (RGBA), PPM (planar) and PGM (grey) sources mixed; strips of 1, 7, 33 and 400 rows (one strip of the
// whole canvas); keep budgets of 0, one image and no limit.  Each run must decode a file exactly once per upload
// the sweep's plan asks for.
// Built by oracle/blend_sweep.mk (needs the reference sources); run by tests/test_gpu_blend_sweep.py on a GPU.
//   blend_sweep_test <dir>     dir: where the image files are written
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

static unsigned g_seed = 777u;
static unsigned rnd() { g_seed = g_seed * 1664525u + 1013904223u; return (g_seed >> 8) & 0xffffff; }

// w×h×3 pixels: a gradient with random discs and a little noise
static std::vector<unsigned char> synth_rgb(int w, int h) {
  std::vector<unsigned char> pix((size_t)w * h * 3);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < 3; ++c)
        pix[((size_t)y * w + x) * 3 + c] = (unsigned char)(40 + (150 * (x + (c + 1) * y)) / (w + 3 * h) + rnd() % 7);
  for (int d = 0; d < (w * h) / 3000; ++d) {
    const int cx = rnd() % w, cy = rnd() % h, r = 3 + rnd() % 20;
    unsigned char col[3] = {(unsigned char)(rnd() & 255), (unsigned char)(rnd() & 255), (unsigned char)(rnd() & 255)};
    for (int y = std::max(0, cy - r); y < std::min(h, cy + r + 1); ++y)
      for (int x = std::max(0, cx - r); x < std::min(w, cx + r + 1); ++x)
        if ((x - cx) * (x - cx) + (y - cy) * (y - cy) <= r * r)
          for (int c = 0; c < 3; ++c) pix[((size_t)y * w + x) * 3 + c] = col[c];
  }
  return pix;
}

// an RGBA PNG (random alpha, which read_img ignores), a PGM of the green channel or a PPM of the pixels
static bool write_file(const std::string& path, const std::vector<unsigned char>& rgb, int w, int h) {
  if (endswith(path.c_str(), ".pgm")) {
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) return false;
    fprintf(f, "P5\n%d %d\n255\n", w, h);
    for (size_t i = 0; i < (size_t)w * h; ++i) fputc(rgb[i * 3 + 1], f);
    fclose(f);
    return true;
  }
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

// The reference's work() tail on read_img's images: blend, crop, write_rgb to `out`.
static void reference_write(const std::vector<View>& views, int W, int H, int bands, Vec2D resolution, Vec2D proj_min,
                            const std::string& out) {
  std::vector<std::unique_ptr<ImageRef>> refs;
  std::unique_ptr<BlenderBase> rb;
  if (bands > 0) rb.reset(new MultiBandBlender{bands}); else rb.reset(new LinearBlender);
  for (auto& v : views) {
    refs.emplace_back(new ImageRef("<memory>"));
    refs.back()->img = new Mat32f(read_img(v.path.c_str()));
    refs.back()->_width = W; refs.back()->_height = H;
    const Homography homo_inv = v.hi;
    Shape2D shp{W, H};
    rb->add_image(v.ul, v.br, *refs.back(), [=](Coor t) -> Vec2D {   // stitcher_image.cc:142-151
      Vec2D c = Vec2D(t.x, t.y) * resolution + proj_min;
      Vec ret = homo_inv.trans(flat::proj2homo(Vec2D(c.x, c.y)));
      if (ret.z < 0) return Vec2D{-10, -10};
      double denom = 1.0 / ret.z;
      return Vec2D{ret.x * denom, ret.y * denom} + shp.center();
    });
  }
  Mat32f res = rb->run();
  write_rgb(out.c_str(), crop(res));
}

static void compare(const Context& ctx, const std::vector<View>& views, int W, int H, int bands,
                    const std::string& dir) {
  config::LAZY_READ = true;
  config::MULTIBAND = bands;
  Vec2D resolution(1.0, 1.0), proj_min(-W / 2.0, -H / 2.0);
  for (const char* ext : {".png", ".ppm"}) {
    const std::string ref_path = dir + "/ref_out" + ext;
    reference_write(views, W, H, bands, resolution, proj_min, ref_path);
    const std::vector<unsigned char> want = file_bytes(ref_path);
    for (size_t keep : {(size_t)0, (size_t)W * H * 4, SIZE_MAX})
      for (int rows : {1, 7, 33, 400}) {
        B200PixelBlender mine(ctx, bands, PANO_PROJ_FLAT, resolution, proj_min);
        for (const View& v : views) mine.add_file(v.ul, v.br, v.path, W, H, v.hi);
        const std::string path = dir + "/b200_out" + ext;
        mine.write_sweep(rows, keep, true, path.c_str());
        const std::vector<unsigned char> got = file_bytes(path);
        const bool same = !want.empty() && want == got;
        const bool once = mine.decodes() == mine.last_sweep_uploads();
        CHECK(same && once, "bands=%d %s keep=%zu rows=%d: %zu reference bytes, %zu from write_sweep; %ld decodes "
              "for %lld uploads", bands, ext, keep, rows, want.size(), got.size(), mine.decodes(),
              mine.last_sweep_uploads());
        if (same && once)
          printf("bands=%d %s keep=%zu rows=%d: %zu file bytes identical, %ld decodes\n", bands, ext, keep, rows,
                 got.size(), mine.decodes());
      }
  }
}

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: blend_sweep_test <dir>\n"); return 2; }
  const std::string dir = argv[1];
  pano_params p;
  pano_params_default(&p);
  set_config(p);
  config::ORDERED_INPUT = false;
  Context ctx(0);
  const int W = 360, H = 270;
  std::vector<View> views;
  for (int k = 0; k < 9; ++k) {
    const char* ext = k % 3 == 0 ? ".png" : k % 3 == 1 ? ".ppm" : ".pgm";
    const std::string path = dir + "/view" + std::to_string(k) + ext;
    if (!write_file(path, synth_rgb(W, H), W, H)) { printf("FAIL: cannot write %s\n", path.c_str()); return 2; }
    const int x = 40 * k, y = 9 * (k % 3) + 70 * (k / 5);
    const double hi[9] = {1, 0, -(double)x, 0, 1, -(double)y, 0, 0, 1};
    views.push_back(View{path, Coor(x, y), Coor(x + W - 1, y + H - 1), Homography(hi)});
  }
  compare(ctx, views, W, H, 0, dir);
  compare(ctx, views, W, H, 5, dir);
  printf(g_fail ? "BLEND SWEEP TEST FAILED (%d)\n" : "BLEND SWEEP TEST OK\n", g_fail);
  return g_fail ? 1 : 0;
}
