// pix_formats_test.cc — compiles the drop-in's file boundary (openpano_b200/host/pano_host_io.hh) against the
// REFERENCE's headers and runs it next to the reference's own file path (oracle/_ref/libopenpano_ref.so: imgio.cc
// with its lodepng and CImg, SIFTDetector, LinearBlender, MultiBandBlender, crop):
//   1. writes PNG files of every colour type with the reference's lodepng (grey, grey+alpha, RGB, RGBA, palette,
//      16-bit RGB and grey) and a PPM and a PGM with CImg's reader in mind, all of one size;
//   2. read_img + SIFTDetector::detect_feature on each file against load_pixels + one detect_batch_rgb8 over all
//      of them (RGBA, planar and grey buffers in one batch);
//   3. LinearBlender (LAZY_READ 1 and 0) and MultiBandBlender on read_img's images against B200PixelBlender on the
//      decoder buffers, windows of 1 and 3;
//   4. write_rgb(crop(mosaic)) to a .png and a .ppm against write_mosaic from the device mosaic, file bytes.
// Coordinates, descriptors and mosaics must be bit-identical.  Built by oracle/pix_formats.mk (needs the reference
// sources); run by tests/test_gpu_pixel_formats.py on a GPU.
//   pix_formats_test <dir>     dir: where the image files are written
#include <cmath>
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

static bool same_desc(const std::vector<Descriptor>& a, const std::vector<Descriptor>& b) {
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); ++i) {
    if (memcmp(&a[i].coor, &b[i].coor, sizeof(Vec2D)) != 0) return false;
    if (a[i].descriptor.size() != b[i].descriptor.size()) return false;
    if (memcmp(a[i].descriptor.data(), b[i].descriptor.data(), a[i].descriptor.size() * sizeof(float)) != 0) return false;
  }
  return true;
}

static bool same_mat(const Mat32f& a, const Mat32f& b) {
  return a.width() == b.width() && a.height() == b.height() &&
         memcmp(a.ptr(), b.ptr(), sizeof(float) * (size_t)a.width() * a.height() * 3) == 0;
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

static unsigned g_seed = 12345u;
static unsigned rnd() { g_seed = g_seed * 1664525u + 1013904223u; return (g_seed >> 8) & 0xffffff; }

// Discs of random colour over a smooth gradient plus a little noise (w×h×3): blob and corner features at every scale.
static std::vector<unsigned char> synth_rgb(int w, int h) {
  std::vector<float> img((size_t)w * h * 3);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < 3; ++c) img[((size_t)y * w + x) * 3 + c] = 60.f + 80.f * (float)(x + (c + 1) * y) / (float)(w + 3 * h);
  for (int d = 0; d < (w * h) / 2500; ++d) {
    const int cx = rnd() % w, cy = rnd() % h, r = 3 + rnd() % 24;
    float col[3];
    for (int c = 0; c < 3; ++c) col[c] = (float)(rnd() % 256);
    for (int y = std::max(0, cy - r); y < std::min(h, cy + r + 1); ++y)
      for (int x = std::max(0, cx - r); x < std::min(w, cx + r + 1); ++x)
        if ((x - cx) * (x - cx) + (y - cy) * (y - cy) <= r * r)
          for (int c = 0; c < 3; ++c) img[((size_t)y * w + x) * 3 + c] = col[c];
  }
  std::vector<unsigned char> pix(img.size());
  for (size_t i = 0; i < img.size(); ++i)
    pix[i] = (unsigned char)std::min(255.f, std::max(0.f, img[i] + (float)((int)(rnd() % 9) - 4)));
  return pix;
}

// A PNG of lodepng colour type `ct` at `bd` bits from w×h×3 pixels: grey takes channel 0, alpha and the low
// byte of 16-bit samples are random, a palette image indexes a 256-colour palette by channel 0.
static bool write_png(const std::string& path, const std::vector<unsigned char>& rgb, int w, int h, LodePNGColorType ct,
                      unsigned bd) {
  lodepng::State st;
  st.encoder.auto_convert = 0;
  st.info_raw.colortype = st.info_png.color.colortype = ct;
  st.info_raw.bitdepth = st.info_png.color.bitdepth = bd;
  std::vector<unsigned char> raw;
  const size_t n = (size_t)w * h;
  if (ct == LCT_PALETTE) {
    for (int k = 0; k < 256; ++k) {
      const unsigned char r = rnd() & 255, g = rnd() & 255, b = rnd() & 255, a = 255;
      lodepng_palette_add(&st.info_png.color, r, g, b, a);
      lodepng_palette_add(&st.info_raw, r, g, b, a);
    }
  }
  for (size_t i = 0; i < n; ++i) {
    std::vector<unsigned char> s;
    if (ct == LCT_GREY || ct == LCT_PALETTE) s = {rgb[i * 3]};
    else if (ct == LCT_GREY_ALPHA) s = {rgb[i * 3], (unsigned char)(rnd() & 255)};
    else if (ct == LCT_RGB) s = {rgb[i * 3], rgb[i * 3 + 1], rgb[i * 3 + 2]};
    else s = {rgb[i * 3], rgb[i * 3 + 1], rgb[i * 3 + 2], (unsigned char)(rnd() & 255)};
    for (unsigned char v : s) {
      raw.push_back(v);
      if (bd == 16) raw.push_back((unsigned char)(rnd() & 255));   // big-endian: the 8-bit value is the high byte
    }
  }
  std::vector<unsigned char> png;
  if (lodepng::encode(png, raw, (unsigned)w, (unsigned)h, st)) return false;
  return lodepng::save_file(png, path) == 0;
}

static bool write_pnm(const std::string& path, const std::vector<unsigned char>& rgb, int w, int h, int ch) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) return false;
  fprintf(f, "%s\n%d %d\n255\n", ch == 3 ? "P6" : "P5", w, h);
  for (size_t i = 0; i < (size_t)w * h; ++i) fwrite(&rgb[i * 3], 1, ch, f);
  fclose(f);
  return true;
}

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
  if (argc < 2) { fprintf(stderr, "usage: pix_formats_test <dir>\n"); return 2; }
  const std::string dir = argv[1];
  pano_params p;
  pano_params_default(&p);
  set_config(p);
  Context ctx(0);

  const int W = 360, H = 270;
  struct File { const char* name; int ct, bd; };   // ct < 0: PNM of -ct channels
  const File files[] = {{"grey.png", LCT_GREY, 8},       {"grey_alpha.png", LCT_GREY_ALPHA, 8}, {"rgb.png", LCT_RGB, 8},
                        {"rgba.png", LCT_RGBA, 8},       {"palette.png", LCT_PALETTE, 8},       {"rgb16.png", LCT_RGB, 16},
                        {"grey16.png", LCT_GREY, 16},    {"rgb.ppm", -3, 8},                    {"grey.pgm", -1, 8}};
  const int n = sizeof(files) / sizeof(files[0]);
  std::vector<Mat32f> mats;
  std::vector<Pixels> px(n);
  for (int k = 0; k < n; ++k) {
    const std::string path = dir + "/" + files[k].name;
    const std::vector<unsigned char> rgb = synth_rgb(W, H);
    const bool ok = files[k].ct >= 0 ? write_png(path, rgb, W, H, (LodePNGColorType)files[k].ct, (unsigned)files[k].bd)
                                     : write_pnm(path, rgb, W, H, -files[k].ct);
    if (!ok) { printf("FAIL: cannot write %s\n", path.c_str()); return 2; }
    mats.push_back(read_img(path.c_str()));                               // the reference's file path
    px[k] = load_pixels(path.c_str());                                    // the drop-in's
    const int want_fmt = files[k].ct >= 0 ? PANO_PIX_RGBA : files[k].ct == -3 ? PANO_PIX_RGB_PLANAR : PANO_PIX_GREY;
    CHECK(px[k].w == W && px[k].h == H && px[k].format == want_fmt, "%s: load_pixels gave %dx%d format %#x",
          files[k].name, px[k].w, px[k].h, px[k].format);
  }

  // 2. SIFT: one batch of every format against detect_feature on each file
  {
    SIFTDetector ref_det;
    B200SIFTDetector det(ctx);
    std::vector<const unsigned char*> ptr(n);
    std::vector<int> w(n, W), h(n, H), fmt(n);
    for (int k = 0; k < n; ++k) { ptr[k] = px[k].ptr(); fmt[k] = px[k].format; }
    auto got = det.detect_batch_rgb8(ptr, w, h, fmt);
    for (int k = 0; k < n; ++k) {
      auto want = ref_det.detect_feature(mats[k]);
      const bool same = same_desc(want, got[k]) && !want.empty();
      CHECK(same, "%s: %zu reference descriptors, %zu from detect_batch_rgb8", files[k].name, want.size(), got[k].size());
      if (same) printf("sift %s: %zu descriptors identical\n", files[k].name, got[k].size());
    }
  }

  // 3. blends: image k shifted by (40k, 9 * (k % 3)) on a flat canvas
  config::ORDERED_INPUT = false;
  Vec2D resolution(1.0, 1.0), proj_min(-W / 2.0, -H / 2.0);
  std::vector<Homography> his(n);
  for (int k = 0; k < n; ++k) {
    const double hi[9] = {1, 0, -40.0 * k, 0, 1, -9.0 * (k % 3), 0, 0, 1};
    his[k] = Homography(hi);
  }
  Mat32f mosaic;
  const int cases[4][2] = {{0, 1}, {0, 0}, {3, 1}, {5, 1}};   // (bands, LAZY_READ)
  for (auto& cs : cases) {
    const int bands = cs[0];
    config::LAZY_READ = cs[1] != 0;
    config::MULTIBAND = bands;
    Mat32f want;
    {
      auto refs = attach(mats);
      std::unique_ptr<BlenderBase> rb;
      if (bands > 0) rb.reset(new MultiBandBlender{bands}); else rb.reset(new LinearBlender);
      for (int k = 0; k < n; ++k) {
        const Homography homo_inv = his[k];
        Shape2D shp{W, H};
        rb->add_image(Coor(40 * k, 9 * (k % 3)), Coor(40 * k + W - 1, 9 * (k % 3) + H - 1), *refs[k],
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
    if (bands == 0 && cs[1]) mosaic = want;
    for (int window : {1, 3}) {
      B200PixelBlender mine(ctx, bands, PANO_PROJ_FLAT, resolution, proj_min, window);
      for (int k = 0; k < n; ++k)
        mine.add_image(Coor(40 * k, 9 * (k % 3)), Coor(40 * k + W - 1, 9 * (k % 3) + H - 1), px[k], his[k]);
      const bool same = same_mat(mine.run(), want);
      CHECK(same, "blend bands=%d lazy=%d window=%d: mosaic differs", bands, cs[1], window);
      if (same) printf("blend bands=%d lazy=%d window=%d: %dx%d identical\n", bands, cs[1], window, want.width(), want.height());
    }
  }

  // 4. crop + write_rgb (main.cc:226-234) against write_mosaic of the same mosaic on the device
  {
    const Mat32f cropped = crop(mosaic);
    void* d = nullptr;
    const size_t bytes = sizeof(float) * (size_t)mosaic.width() * mosaic.height() * 3;
    ctx.check(pano_dev_alloc(ctx.get(), bytes, &d));
    ctx.check(pano_dev_upload(ctx.get(), d, mosaic.ptr(), bytes));
    for (const char* ext : {".png", ".ppm"}) {
      const std::string ref_path = dir + "/ref_out" + ext, mine_path = dir + "/b200_out" + ext;
      write_rgb(ref_path.c_str(), cropped);
      write_mosaic(ctx, (const float*)d, mosaic.width(), mosaic.height(), true, mine_path.c_str());
      const std::vector<unsigned char> a = file_bytes(ref_path), b = file_bytes(mine_path);
      const bool same = !a.empty() && a == b;
      CHECK(same, "write %s: %zu reference bytes, %zu from write_mosaic", ext, a.size(), b.size());
      if (same) printf("write %s: %dx%d, %zu file bytes identical\n", ext, cropped.width(), cropped.height(), a.size());
    }
    ctx.check(pano_dev_free(ctx.get(), d));
  }
  printf(g_fail ? "PIX FORMATS TEST FAILED (%d)\n" : "PIX FORMATS TEST OK\n", g_fail);
  return g_fail ? 1 : 0;
}
