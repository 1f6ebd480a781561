// adaptor_test.cc — compiles the drop-in's C++ host (openpano_b200/host/pano_host.hh) against
// the REFERENCE's headers and runs every adaptor next to the reference class it replaces:
//   B200SIFTDetector   vs SIFTDetector          (feature/feature.hh:42-57)
//   B200PairMatcher    vs FeatureMatcher        (feature/matcher.hh:27-38, the exact rule)
//   B200Blender        vs LinearBlender / MultiBandBlender (stitch/blender.hh, multiband.hh)
//   B200CylinderWarper vs CylinderWarper        (stitch/warp.hh:41-66)
//   B200Stitcher::build  = the three stages chained as Stitcher::build() chains them
// Results must be bit-identical.  The reference classes come from oracle/_ref/libopenpano_ref.so
// (the reference's own TUs, parity flags); the engine from openpano_b200/libpano_b200.so.
// Built by oracle/Makefile (needs the reference sources); run by tests/test_gpu_adaptors.py on a GPU.
//   adaptor_test <stack.bin>     stack.bin: int32 n, w, h, then n*h*w*3 float32, then per image
//                                 int32 x0,y0,x1,y1 + float64 homo_inv[9], then float64 res, min_x, min_y
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#include "pano_host.hh"
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
  return a.width() == b.width() && a.height() == b.height() && a.channels() == b.channels() &&
         memcmp(a.ptr(), b.ptr(), sizeof(float) * (size_t)a.width() * a.height() * a.channels()) == 0;
}

struct Item { int x0, y0, x1, y1; double hi[9]; };

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: adaptor_test stack.bin\n"); return 2; }
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
  std::vector<Item> items(n);
  for (int k = 0; k < n; ++k) {
    if (fread(&items[k].x0, 4, 4, f) != 4) return 2;
    if (fread(items[k].hi, 8, 9, f) != 9) return 2;
  }
  double geo[3];
  if (fread(geo, 8, 3, f) != 3) return 2;
  fclose(f);

  pano_params p;
  pano_params_default(&p);
  set_config(p);
  Context ctx(0);

  // ---- features
  SIFTDetector ref_det;
  B200SIFTDetector det(ctx);
  std::vector<std::vector<Descriptor>> ref_feats(n);
  size_t total = 0;
  for (int k = 0; k < n; ++k) {
    ref_feats[k] = ref_det.detect_feature(imgs[k]);                    // reference: scaling in the base class
    auto mine = static_cast<const FeatureDetector&>(det).detect_feature(imgs[k]);   // same base-class entry, our virtual
    CHECK(same_desc(ref_feats[k], mine), "detect_feature differs on image %d (%zu vs %zu)", k, ref_feats[k].size(), mine.size());
    auto raw_ref = ref_det.do_detect_feature(imgs[k]);
    auto raw = det.do_detect_feature(imgs[k]);
    CHECK(same_desc(raw_ref, raw), "do_detect_feature differs on image %d", k);
    total += mine.size();
  }
  std::vector<const Mat32f*> ptrs;
  for (auto& m : imgs) ptrs.push_back(&m);
  pano_featureset* fs = nullptr;
  auto batch = det.detect_batch(ptrs, &fs);
  for (int k = 0; k < n; ++k) CHECK(same_desc(ref_feats[k], batch[k]), "detect_batch differs on image %d", k);
  printf("features: %zu descriptors over %d images\n", total, n);

  // ---- matching (both constructor shapes)
  {
    B200PairMatcher from_dev(ctx, fs), from_host(ctx, ref_feats);
    size_t nm = 0;
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) {
        if (i == j) continue;
        MatchData want = FeatureMatcher(ref_feats[i], ref_feats[j]).match();
        MatchData a = from_dev.match(i, j), b = from_host.match(i, j);
        CHECK(want.data == a.data, "match(%d,%d) from device descriptors: %d vs %d", i, j, want.size(), a.size());
        CHECK(want.data == b.data, "match(%d,%d) from host descriptors: %d vs %d", i, j, want.size(), b.size());
        nm += want.size();
      }
    printf("matching: %zu pairs over %d ordered image pairs\n", nm, n * (n - 1));
  }
  pano_featureset_free(fs);

  // ---- blenders (LAZY_READ on and off, linear and 3 bands)
  Vec2D resolution(geo[0], geo[0]), proj_min(geo[1], geo[2]);
  for (int bands : {0, 3})
    for (int lazy : {1, 0}) {
      config::LAZY_READ = lazy != 0;
      config::MULTIBAND = bands;
      std::vector<std::unique_ptr<ImageRef>> refs;
      for (int k = 0; k < n; ++k) {
        refs.emplace_back(new ImageRef("<memory>"));
        refs.back()->img = new Mat32f(imgs[k].clone());
        refs.back()->_width = w; refs.back()->_height = h;
      }
      std::unique_ptr<BlenderBase> rb;
      if (bands > 0) rb.reset(new MultiBandBlender{bands}); else rb.reset(new LinearBlender);
      B200Blender mine(ctx, bands, PANO_PROJ_FLAT, resolution, proj_min);
      for (int k = 0; k < n; ++k) {
        Homography homo_inv(items[k].hi);
        Shape2D shp{w, h};
        rb->add_image(Coor(items[k].x0, items[k].y0), Coor(items[k].x1, items[k].y1), *refs[k],
                      [=](Coor t) -> Vec2D {                           // stitcher_image.cc:142-151
                        Vec2D c = Vec2D(t.x, t.y) * resolution + proj_min;
                        Vec homo = flat::proj2homo(Vec2D(c.x, c.y));
                        Vec ret = homo_inv.trans(homo);
                        if (ret.z < 0) return Vec2D{-10, -10};
                        double denom = 1.0 / ret.z;
                        return Vec2D{ret.x * denom, ret.y * denom} + shp.center();
                      });
        mine.add_image(Coor(items[k].x0, items[k].y0), Coor(items[k].x1, items[k].y1), *refs[k], homo_inv);
      }
      // engine first: with LAZY_READ the reference's run() releases every image after its single use
      // (blender.cc:47,63, multiband.cc:27,49; load() is a no-op while the Mat is still attached)
      Mat32f got = mine.run();
      Mat32f want = rb->run();
      CHECK(same_mat(want, got), "blend bands=%d lazy=%d differs", bands, lazy);
      printf("blend bands=%d lazy=%d: %dx%d ok\n", bands, lazy, got.width(), got.height());
    }
  config::LAZY_READ = true; config::MULTIBAND = 0;

  // ---- cylinder warp
  {
    Mat32f a = imgs[0].clone(), b = imgs[0].clone();
    std::vector<Vec2D> ka{Vec2D(10.5, -20.25), Vec2D(-100, 50), Vec2D(0, 0)}, kb = ka;
    CylinderWarper(1.0).warp(a, ka);
    B200CylinderWarper(ctx, 1.0).warp(b, kb);
    CHECK(same_mat(a, b), "cylinder warp image differs");
    CHECK(memcmp(ka.data(), kb.data(), sizeof(Vec2D) * ka.size()) == 0, "cylinder warp keypoints differ");
    printf("cylinder warp: %dx%d ok\n", b.width(), b.height());
  }

  // ---- the chained hot path of Stitcher::build()
  {
    config::ORDERED_INPUT = true; config::LAZY_READ = false; config::MULTIBAND = 0;
    std::vector<ImageRef> refs;
    refs.reserve(n);
    for (int k = 0; k < n; ++k) {
      refs.emplace_back("<memory>");
      refs.back().img = new Mat32f(imgs[k].clone());
      refs.back()._width = w; refs.back()._height = h;
    }
    StitchGeometry g;
    g.resolution = resolution; g.proj_min = proj_min;
    for (int k = 0; k < n; ++k) {
      g.upper_left.emplace_back(items[k].x0, items[k].y0);
      g.bottom_right.emplace_back(items[k].x1, items[k].y1);
      g.homo_inv.emplace_back(items[k].hi);
    }
    B200Stitcher st(ctx);
    Mat32f mosaic = st.build(refs, g);
    for (int k = 0; k < n; ++k) CHECK(same_desc(ref_feats[k], st.feats[k]), "B200Stitcher features differ on image %d", k);
    for (size_t t = 0; t < st.pairs.size(); ++t) {
      MatchData want = FeatureMatcher(ref_feats[st.pairs[t].first], ref_feats[st.pairs[t].second]).match();
      CHECK(want.data == st.matches[t].data, "B200Stitcher match %zu differs", t);
    }
    LinearBlender lb;
    std::vector<std::unique_ptr<ImageRef>> keep;
    for (int k = 0; k < n; ++k) {
      keep.emplace_back(new ImageRef("<memory>"));
      keep.back()->img = new Mat32f(imgs[k].clone());
      keep.back()->_width = w; keep.back()->_height = h;
      Homography homo_inv(items[k].hi);
      Shape2D shp{w, h};
      lb.add_image(g.upper_left[k], g.bottom_right[k], *keep[k], [=](Coor t) -> Vec2D {
        Vec2D c = Vec2D(t.x, t.y) * resolution + proj_min;
        Vec ret = homo_inv.trans(flat::proj2homo(Vec2D(c.x, c.y)));
        if (ret.z < 0) return Vec2D{-10, -10};
        double denom = 1.0 / ret.z;
        return Vec2D{ret.x * denom, ret.y * denom} + shp.center();
      });
    }
    Mat32f want = lb.run();
    CHECK(same_mat(want, mosaic), "B200Stitcher mosaic differs");
    printf("B200Stitcher::build: %zu match lists, mosaic %dx%d ok\n", st.matches.size(), mosaic.width(), mosaic.height());
  }

  printf(g_fail ? "ADAPTOR TEST FAILED (%d)\n" : "ADAPTOR TEST OK\n", g_fail);
  return g_fail ? 1 : 0;
}
