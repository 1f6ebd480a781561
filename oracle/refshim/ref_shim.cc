// ref_shim.cc — exposes the REFERENCE's own hot-path classes through the
// checker API (oracle/oracle_api.h, prefix ref_).  TEST INFRASTRUCTURE ONLY.
//
// This file contains no algorithm: every call lands in a translation unit that
// is compiled, unmodified, from the reference's src/ by oracle/Makefile.  The
// only stand-ins are lib/matrix.cc (needs Eigen, absent here: see
// matrix_standin.cc) and a syntactic Eigen/Dense stub so lib/imgproc.cc compiles
// (its two Eigen functions are off the hot path and are never called).
// lib/imgio.cc is built with -DDISABLE_JPEG (CImg's native PNM reader/writer and
// the vendored lodepng need no external library); ref_imgio.cc drives it.
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>
#include <cmath>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "lib/config.hh"
#include "lib/timer.hh"
#include "lib/mat.h"
#include "lib/imgproc.hh"
#include "feature/feature.hh"
#include "feature/dog.hh"
#include "feature/extrema.hh"
#include "feature/orientation.hh"
#include "feature/sift.hh"
#include "feature/matcher.hh"
#include "stitch/warp.hh"
#include "stitch/blender.hh"
#include "stitch/multiband.hh"
#include "stitch/projection.hh"
#include "stitch/homography.hh"
#define private public          // get_inliers / ransac_inlier_thres are private members of TransformEstimation
#include "stitch/transform_estimate.hh"
#undef private

#include "../oracle_api.h"

using namespace pano;

namespace {

void apply_params(const pano_params* p) {
  using namespace config;
  CYLINDER = false; TRANS = false; CROP = true; ESTIMATE_CAMERA = true; STRAIGHTEN = true;
  FOCAL_LENGTH = p->focal_length;
  MAX_OUTPUT_SIZE = p->max_output_size;
  ORDERED_INPUT = p->ordered_input != 0;
  LAZY_READ = p->lazy_read != 0;
  SIFT_WORKING_SIZE = p->sift_working_size;
  NUM_OCTAVE = p->num_octave;
  NUM_SCALE = p->num_scale;
  SCALE_FACTOR = p->scale_factor;
  GAUSS_SIGMA = p->gauss_sigma;
  GAUSS_WINDOW_FACTOR = p->gauss_window_factor;
  JUDGE_EXTREMA_DIFF_THRES = p->judge_extrema_diff_thres;
  CONTRAST_THRES = p->contrast_thres;
  PRE_COLOR_THRES = p->pre_color_thres;
  EDGE_RATIO = p->edge_ratio;
  CALC_OFFSET_DEPTH = p->calc_offset_depth;
  OFFSET_THRES = p->offset_thres;
  ORI_RADIUS = p->ori_radius;
  ORI_HIST_SMOOTH_COUNT = p->ori_hist_smooth_count;
  DESC_HIST_SCALE_FACTOR = p->desc_hist_scale_factor;
  DESC_INT_FACTOR = p->desc_int_factor;
  MATCH_REJECT_NEXT_RATIO = p->match_reject_next_ratio;
  MULTIBAND = p->multiband;
  RANSAC_ITERATIONS = 1500; RANSAC_INLIER_THRES = 3.5;
  INLIER_IN_MATCH_RATIO = 0.1f; INLIER_IN_POINTS_RATIO = 0.04f;
  SLOPE_PLAIN = 8e-3f; LM_LAMBDA = 5; MULTIPASS_BA = 1;
}

Mat32f wrap_rgb(const float* rgb, int w, int h) {
  Mat32f m(h, w, 3);
  memcpy(m.ptr(), rgb, sizeof(float) * (size_t)w * h * 3);
  return m;
}

// get_local_raw_extrema is protected in the reference.
struct ExtremaProbe : public ExtremaDetector {
  explicit ExtremaProbe(const DOGSpace& d) : ExtremaDetector(d) {}
  std::vector<Coor> raw(int pyr, int scale) const { return get_local_raw_extrema(pyr, scale); }
};

pano_sspoint to_pod(const SSPoint& s) {
  pano_sspoint o;
  o.x = s.coor.x; o.y = s.coor.y;
  o.real_x = s.real_coor.x; o.real_y = s.real_coor.y;
  o.pyr_id = s.pyr_id; o.scale_id = s.scale_id;
  o.dir = s.dir; o.scale_factor = s.scale_factor;
  return o;
}

}  // namespace

struct ref_sift {
  int in_w, in_h;
  Mat32f working;
  std::unique_ptr<ScaleSpace> ss;
  std::unique_ptr<DOGSpace> dog;
  std::vector<pano_sspoint> raw, refined, oriented;
  std::vector<Descriptor> desc;
};

extern "C" {

int ref_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

// Mirrors SIFTDetector::do_detect_feature (feature/feature.cc:31-47) statement by
// statement, keeping each intermediate alive.
ref_sift* ref_sift_run(const float* rgb, int w, int h, const pano_params* p) {
  apply_params(p);
  ref_sift* s = new ref_sift;
  s->in_w = w; s->in_h = h;
  Mat32f mat = wrap_rgb(rgb, w, h);
  float ratio = config::SIFT_WORKING_SIZE * 2.0f / (mat.width() + mat.height());
  s->working = Mat32f(mat.rows() * ratio, mat.cols() * ratio, 3);
  resize(mat, s->working);
  s->ss.reset(new ScaleSpace(s->working, config::NUM_OCTAVE, config::NUM_SCALE));
  s->dog.reset(new DOGSpace(*s->ss));
  ExtremaProbe ex(*s->dog);
  for (int i = 0; i < s->dog->noctave; ++i)
    for (int j = 1; j < s->dog->nscale - 2; ++j)
      for (auto& c : ex.raw(i, j)) {
        pano_sspoint q; memset(&q, 0, sizeof(q));
        q.x = c.x; q.y = c.y; q.pyr_id = i; q.scale_id = j;
        s->raw.push_back(q);
      }
  auto keyp = ex.get_extrema();
  for (auto& k : keyp) { k.dir = 0; s->refined.push_back(to_pod(k)); }
  OrientationAssign ort(*s->dog, *s->ss, keyp);
  keyp = ort.work();
  for (auto& k : keyp) s->oriented.push_back(to_pod(k));
  SIFT sift(*s->ss, keyp);
  s->desc = sift.get_descriptor();
  // FeatureDetector::detect_feature (feature.cc:20-28)
  for (auto& d : s->desc) {
    d.coor.x = (d.coor.x - 0.5) * w;
    d.coor.y = (d.coor.y - 0.5) * h;
  }
  return s;
}

void ref_sift_working_size(const ref_sift* s, int* w0, int* h0) {
  *w0 = s->working.width(); *h0 = s->working.height();
}

int ref_sift_octave_size(const ref_sift* s, int o, int* w, int* h) {
  if (o < 0 || o >= s->ss->noctave) return -1;
  *w = s->ss->pyramids[o].w; *h = s->ss->pyramids[o].h;
  return 0;
}

int ref_sift_plane(const ref_sift* s, int kind, int o, int level, float* out) {
  const Mat32f* m = nullptr;
  if (kind == 0) m = &s->working;
  else {
    if (o < 0 || o >= s->ss->noctave) return -1;
    const GaussianPyramid& py = s->ss->pyramids[o];
    int ns = py.get_len();
    if (kind == 1) { if (level < 0 || level >= ns) return -1; m = &py.get(level); }
    else if (kind == 2) { if (level < 0 || level >= ns - 1) return -1; m = &s->dog->dogs[o][level]; }
    else if (kind == 3) { if (level < 1 || level >= ns) return -1; m = &py.get_mag(level); }
    else if (kind == 4) { if (level < 1 || level >= ns) return -1; m = &py.get_ort(level); }
    else return -1;
  }
  memcpy(out, m->ptr(), sizeof(float) * (size_t)m->pixels() * m->channels());
  return 0;
}

int ref_sift_points(const ref_sift* s, int stage, int cap, pano_sspoint* out) {
  const std::vector<pano_sspoint>& v = stage == 0 ? s->raw : stage == 1 ? s->refined : s->oriented;
  int n = (int)v.size();
  for (int i = 0; i < n && i < cap; ++i) out[i] = v[i];
  return n;
}

int ref_sift_descriptors(const ref_sift* s, int cap, double* coor, float* desc) {
  int n = (int)s->desc.size();
  for (int i = 0; i < n && i < cap; ++i) {
    if (coor) { coor[2 * i] = s->desc[i].coor.x; coor[2 * i + 1] = s->desc[i].coor.y; }
    if (desc) memcpy(desc + (size_t)128 * i, s->desc[i].descriptor.data(), 128 * sizeof(float));
  }
  return n;
}

void ref_sift_free(ref_sift* s) { delete s; }

int ref_sift_detect(const float* rgb, int w, int h, const pano_params* p, int cap,
                    double* coor, float* desc) {
  apply_params(p);
  SIFTDetector det;
  Mat32f mat = wrap_rgb(rgb, w, h);
  auto d = det.detect_feature(mat);
  int n = (int)d.size();
  if (n > cap) return -1;
  for (int i = 0; i < n; ++i) {
    if (coor) { coor[2 * i] = d[i].coor.x; coor[2 * i + 1] = d[i].coor.y; }
    if (desc) memcpy(desc + (size_t)128 * i, d[i].descriptor.data(), 128 * sizeof(float));
  }
  return n;
}

int ref_match(const float* a, int n, const float* b, int m, const pano_params* p,
              int* pairs, int* npairs) {
  apply_params(p);
  std::vector<Descriptor> f1(n), f2(m);
  for (int i = 0; i < n; ++i) f1[i].descriptor.assign(a + (size_t)128 * i, a + (size_t)128 * (i + 1));
  for (int i = 0; i < m; ++i) f2[i].descriptor.assign(b + (size_t)128 * i, b + (size_t)128 * (i + 1));
  FeatureMatcher fm(f1, f2);
  MatchData md = fm.match();
  // omp critical push order is arbitrary with >1 thread: canonical order is the
  // single-thread one, ascending index of the smaller set (SURVEY §8a a16).
  bool rev = n > m;
  std::sort(md.data.begin(), md.data.end(), [rev](const std::pair<int,int>& x, const std::pair<int,int>& y) {
    return rev ? x.second < y.second : x.first < y.first; });
  *npairs = md.size();
  for (int i = 0; i < md.size(); ++i) { pairs[2 * i] = md.data[i].first; pairs[2 * i + 1] = md.data[i].second; }
  return 0;
}

// CylinderWarper::warp(Shape2D&, kpts) (warp.hh:54-57)
int ref_cyl_warp_shape(int w, int h, double h_factor, const pano_params* p,
                       int* ow, int* oh, double* offx, double* offy) {
  apply_params(p);
  // get_projector is protected; reproduce its two lines via a subclass
  struct W : CylinderWarper { W(double f) : CylinderWarper(f) {}
    CylinderProject proj(int w, int h) const { return get_projector(w, h); } } cw(h_factor);
  Shape2D shape{w, h};
  std::vector<Vec2D> none;
  Vec2D off = cw.proj(w, h).project(shape, none);
  *ow = shape.w; *oh = shape.h; *offx = off.x; *offy = off.y;
  return 0;
}

int ref_cyl_warp(const float* rgb, int w, int h, double h_factor, const pano_params* p,
                 float* out, int ow, int oh, double* kpts, int nk) {
  apply_params(p);
  CylinderWarper cw(h_factor);
  Mat32f mat = wrap_rgb(rgb, w, h);
  std::vector<Vec2D> pts;
  for (int i = 0; i < nk; ++i) pts.emplace_back(kpts[2 * i], kpts[2 * i + 1]);
  cw.warp(mat, pts);
  if (mat.width() != ow || mat.height() != oh) return -1;
  memcpy(out, mat.ptr(), sizeof(float) * (size_t)ow * oh * 3);
  for (int i = 0; i < nk; ++i) { kpts[2 * i] = pts[i].x; kpts[2 * i + 1] = pts[i].y; }
  return 0;
}

// Drives LinearBlender / MultiBandBlender exactly as ConnectedImages::blend does
// (stitch/stitcher_image.cc:132-154); the lambda below is that file's :142-151.
int ref_blend(int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
              const pano_params* p, float* out, int ow, int oh) {
  apply_params(p);
  std::vector<std::unique_ptr<ImageRef>> refs;
  for (int k = 0; k < n; ++k) {
    refs.emplace_back(new ImageRef("<memory>"));
    refs.back()->img = new Mat32f(wrap_rgb(imgs[k].rgb_hwc, imgs[k].w, imgs[k].h));
    refs.back()->_width = imgs[k].w;
    refs.back()->_height = imgs[k].h;
  }
  std::unique_ptr<BlenderBase> blender;
  if (bands > 0) blender.reset(new MultiBandBlender{bands});
  else blender.reset(new LinearBlender);
  proj2homo_t proj2homo = g->projection == PANO_PROJ_FLAT ? flat::proj2homo
                        : g->projection == PANO_PROJ_CYLINDRICAL ? cylindrical::proj2homo
                        : spherical::proj2homo;
  Vec2D resolution(g->res_x, g->res_y), proj_min(g->proj_min_x, g->proj_min_y);
  for (int k = 0; k < n; ++k) {
    Homography homo_inv(imgs[k].homo_inv);
    ImageRef* ir = refs[k].get();
    Shape2D shp{imgs[k].w, imgs[k].h};
    blender->add_image(Coor(imgs[k].x0, imgs[k].y0), Coor(imgs[k].x1, imgs[k].y1), *ir,
        [=](Coor t) -> Vec2D {
          Vec2D c = Vec2D(t.x, t.y) * resolution + proj_min;
          Vec homo = proj2homo(Vec2D(c.x, c.y));
          Vec ret = homo_inv.trans(homo);
          if (ret.z < 0)
            return Vec2D{-10, -10};
          double denom = 1.0 / ret.z;
          return Vec2D{ret.x*denom, ret.y*denom} + shp.center();
        });
  }
  Mat32f res = blender->run();
  if (res.width() != ow || res.height() != oh) return -1;
  memcpy(out, res.ptr(), sizeof(float) * (size_t)ow * oh * 3);
  return 0;
}


// The hot path as Stitcher::build() drives it: calc_feature (stitcherbase.cc:9-27,
// omp over images), linear/pairwise match (stitcher.cc:96-136, omp over pairs, the
// FLANN PairWiseMatcher unless use_flann == 0), ConnectedImages::blend's blender
// (stitcher_image.cc:132-154).  RANSAC / camera estimation are host geometry
// outside the hot path and are replaced by caller-supplied homographies.
int ref_hotpath(int n, const float* const* rgb, const int* w, const int* h, int n_pairs, const int* ij,
                int use_flann, const pano_blend_image* bimgs, const pano_blend_geom* g, int bands,
                const pano_params* p, float* out, int ow, int oh, int* n_feat, int* n_match, double* seconds) {
  apply_params(p);
  Timer t0;
  std::vector<std::vector<Descriptor>> feats(n);
  std::unique_ptr<FeatureDetector> feature_det(new SIFTDetector);
#pragma omp parallel for schedule(dynamic)
  for (int k = 0; k < n; ++k) {
    Mat32f img = wrap_rgb(rgb[k], w[k], h[k]);
    feats[k] = feature_det->detect_feature(img);
  }
  for (int k = 0; k < n; ++k) { n_feat[k] = (int)feats[k].size(); if (!n_feat[k]) return -5; }
  seconds[0] = t0.duration();
  Timer t1;
  if (use_flann) {
    PairWiseMatcher pwmatcher(feats);
#pragma omp parallel for schedule(dynamic)
    for (int k = 0; k < n_pairs; ++k) n_match[k] = pwmatcher.match(ij[2 * k], ij[2 * k + 1]).size();
  } else {
    // FeatureMatcher parallelises internally (matcher.cc:32)
    for (int k = 0; k < n_pairs; ++k) {
      FeatureMatcher fm(feats[ij[2 * k]], feats[ij[2 * k + 1]]);
      n_match[k] = fm.match().size();
    }
  }
  seconds[1] = t1.duration();
  Timer t2;
  int rc = ref_blend(n, bimgs, g, bands, p, out, ow, oh);
  seconds[2] = t2.duration();
  return rc;
}

// TransformEstimation::get_inliers itself (transform_estimate.cc:132-148), driven like the loop
// of get_transform (:68-85) with caller-supplied hypotheses.
int ref_ransac_score(int n_match, const double* kp1_xy, const double* kp2_xy, int n_hyp, const double* homos,
                     float inlier_thres, int* hyp_counts, int* best_hyp, int* best_count, unsigned char* inlier_flags) {
  MatchData md;
  std::vector<Vec2D> kp1(n_match), kp2(n_match);
  for (int i = 0; i < n_match; ++i) {
    md.data.emplace_back(i, i);
    kp1[i] = Vec2D(kp1_xy[2 * i], kp1_xy[2 * i + 1]);
    kp2[i] = Vec2D(kp2_xy[2 * i], kp2_xy[2 * i + 1]);
  }
  *best_hyp = -1; *best_count = 0;
  if (inlier_flags) memset(inlier_flags, 0, n_match);
  if (n_match < 8) return n_hyp > 0 ? -1 : 0;          // the constructor leaves f2_homo_coor empty below 8 matches
  TransformEstimation te(md, kp1, kp2, Shape2D{800, 800}, Shape2D{800, 800});
  te.ransac_inlier_thres = inlier_thres;
  int maxcnt = -1;
  for (int k = 0; k < n_hyp; ++k) {
    double arr[9];
    memcpy(arr, homos + 9 * (size_t)k, sizeof(arr));
    int cnt = (int)te.get_inliers(Homography(arr)).size();
    if (hyp_counts) hyp_counts[k] = cnt;
    if (update_max(maxcnt, cnt)) *best_hyp = k;
  }
  if (*best_hyp >= 0) {
    double arr[9];
    memcpy(arr, homos + 9 * (size_t)*best_hyp, sizeof(arr));
    std::vector<int> in = te.get_inliers(Homography(arr));
    *best_count = (int)in.size();
    if (inlier_flags) for (int i : in) inlier_flags[i] = 1;
  }
  return 0;
}

}  // extern "C"
