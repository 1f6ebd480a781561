// pano_host.hh — the C++ host side of the drop-in: adaptor classes that a maintainer adds to
// the reference tree (INTEGRATION.md).  They derive from / mirror the reference's own seams
//   FeatureDetector      feature/feature.hh:42-52
//   PairWiseMatcher      feature/matcher.hh:40-67  (same constructor shape and match(i, j))
//   BlenderBase          stitch/blender.hh:14-59
//   CylinderWarper       stitch/warp.hh:41-66
//   planet()             main.cc:294-331, the little-planet view: b200_planet
//   the LM loop of IncrementalBundleAdjuster::optimize (stitch/incremental_bundle_adjuster.cc:117-169):
//                        calcError and get_param_update's J / J^T J / b, B200BundleAdjusterStep
// and forward to the C ABI of libpano_b200.so (include/pano_b200.h).  Header-only; compiles
// against the reference's headers (-I <reference>/src) with the reference's own flags.
// tests/adaptor/adaptor_test.cc builds these against the reference tree and checks them
// against the reference classes they replace, bit for bit.
#pragma once
#include <algorithm>
#include <cstring>
#include <functional>
#include <memory>
#include <vector>

#include "pano_b200.h"

#include "lib/config.hh"
#include "lib/mat.h"
#include "lib/geometry.hh"
#include "lib/debugutils.hh"
#include "feature/feature.hh"
#include "feature/matcher.hh"
#include "stitch/blender.hh"
#include "stitch/warp.hh"
#include "stitch/homography.hh"
#include "stitch/camera.hh"
#include "stitch/match_info.hh"
#include "stitch/stitcher_image.hh"
#include "lib/imgproc.hh"

namespace pano_b200 {

// lib/config.hh:24-68 -> the POD snapshot every engine call takes
inline pano_params snapshot_params() {
  using namespace config;
  pano_params p;
  pano_params_default(&p);
  p.sift_working_size = SIFT_WORKING_SIZE; p.num_octave = NUM_OCTAVE; p.num_scale = NUM_SCALE;
  p.scale_factor = SCALE_FACTOR; p.gauss_sigma = GAUSS_SIGMA; p.gauss_window_factor = GAUSS_WINDOW_FACTOR;
  p.judge_extrema_diff_thres = JUDGE_EXTREMA_DIFF_THRES; p.contrast_thres = CONTRAST_THRES;
  p.pre_color_thres = PRE_COLOR_THRES; p.edge_ratio = EDGE_RATIO; p.calc_offset_depth = CALC_OFFSET_DEPTH;
  p.offset_thres = OFFSET_THRES; p.ori_radius = ORI_RADIUS; p.ori_hist_smooth_count = ORI_HIST_SMOOTH_COUNT;
  p.desc_hist_scale_factor = DESC_HIST_SCALE_FACTOR; p.desc_int_factor = DESC_INT_FACTOR;
  p.match_reject_next_ratio = MATCH_REJECT_NEXT_RATIO; p.focal_length = FOCAL_LENGTH;
  p.ordered_input = ORDERED_INPUT; p.lazy_read = LAZY_READ; p.multiband = MULTIBAND;
  p.max_output_size = MAX_OUTPUT_SIZE;
  return p;
}

// One engine context per process (main.cc creates it after init_config()).
class Context {
 public:
  explicit Context(int device = 0) {
    if (pano_create(&ctx_, device, nullptr) != 0) error_exit(pano_last_error(nullptr));
  }
  ~Context() { pano_destroy(ctx_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  pano_ctx* get() const { return ctx_; }
  void check(int rc) const { if (rc != 0) error_exit(pano_last_error(ctx_)); }   // the reference's error convention
 private:
  pano_ctx* ctx_ = nullptr;
};

// Loads refs `window` at a time, hands each window to add(first, count, srcs) and releases it before the next window
// is loaded, so at most one window of Mat32f is resident on the host.  Mat32f storage is pageable: the streams stage
// it before add returns.
template <class Add>
inline void add_windows(const std::vector<pano::ImageRef*>& refs, int window, Add add) {
  const int n = (int)refs.size();
  for (int k0 = 0; k0 < n; k0 += window) {
    const int k1 = std::min(n, k0 + window);
    std::vector<const void*> src;
    for (int k = k0; k < k1; ++k) {
      refs[k]->load();
      src.push_back(refs[k]->img->ptr());
    }
    add(k0, k1 - k0, src.data());
    for (int k = k0; k < k1; ++k) refs[k]->release();
  }
}

// The blend geometry of a BlenderBase: the projection, its resolution and the range's minimum
inline pano_blend_geom blend_geom(int projection, Vec2D resolution, Vec2D proj_min) {
  pano_blend_geom g;
  g.projection = projection; g.res_x = resolution.x; g.res_y = resolution.y;
  g.proj_min_x = proj_min.x; g.proj_min_y = proj_min.y;
  return g;
}

// ---- features: a FeatureDetector (feature.hh:42-52).  do_detect_feature returns real_coor in
// [0,1) exactly as SIFTDetector::do_detect_feature does; the non-virtual detect_feature of the
// base class then applies its own scaling (feature.cc:20-28).
class B200SIFTDetector : public pano::FeatureDetector {
 public:
  explicit B200SIFTDetector(const Context& c) : c_(c) {}
  std::vector<pano::Descriptor> do_detect_feature(const Mat32f& img) const override {
    pano_params p = snapshot_params();
    pano_featureset* fs = nullptr;
    c_.check(pano_sift_detect(c_.get(), img.ptr(), img.width(), img.height(), &p, &fs));
    auto out = unpack(fs, 0, /*real=*/true);
    pano_featureset_free(fs);
    return out;
  }
  // calc_feature()'s loop over images (stitcherbase.cc:14-17) as ONE batched call; descriptors
  // stay on the device in *keep for B200PairMatcher.  Coordinates come back already scaled
  // ((c - 0.5) * w), like detect_feature's.
  std::vector<std::vector<pano::Descriptor>> detect_batch(const std::vector<const Mat32f*>& imgs,
                                                          pano_featureset** keep = nullptr) const {
    const int n = (int)imgs.size();
    std::vector<const float*> ptr(n);
    std::vector<int> w(n), h(n);
    for (int k = 0; k < n; ++k) { ptr[k] = imgs[k]->ptr(); w[k] = imgs[k]->width(); h[k] = imgs[k]->height(); }
    pano_params p = snapshot_params();
    pano_featureset* fs = nullptr;
    c_.check(pano_sift_detect_batch(c_.get(), n, ptr.data(), w.data(), h.data(), &p, &fs));
    return unpack_batch(fs, n, keep);
  }
  // detect_batch for callers that decode the files themselves: pix[k] is h[k]×w[k]×channels[k] interleaved
  // 8-bit pixels in host memory (channels 1 or 3, what read_img converts, lib/imgio.cc:72-88), or a decoder's
  // own buffer with its PANO_PIX_* format as channels[k] (pano_host_io.hh's load_pixels).  Returns what
  // detect_batch returns on read_img's Mat32f of the same pixels, without building those images.
  std::vector<std::vector<pano::Descriptor>> detect_batch_rgb8(const std::vector<const unsigned char*>& pix,
                                                               const std::vector<int>& w, const std::vector<int>& h,
                                                               const std::vector<int>& channels,
                                                               pano_featureset** keep = nullptr) const {
    const int n = (int)pix.size();
    if ((int)w.size() != n || (int)h.size() != n || (int)channels.size() != n)
      error_exit("B200SIFTDetector::detect_batch_rgb8: pix, w, h and channels differ in length");
    pano_params p = snapshot_params();
    pano_featureset* fs = nullptr;
    c_.check(pano_sift_detect_batch_rgb8(c_.get(), n, pix.data(), w.data(), h.data(), channels.data(), &p, &fs));
    return unpack_batch(fs, n, keep);
  }
  // calc_feature()'s LAZY_READ branch (stitcherbase.cc:14-19): the images are loaded `window` at a time, handed to a
  // pano_sift_stream and released before the next window is loaded, so at most one window of Mat32f is resident on
  // the host and two on the device.  Returns detect_batch's descriptors on the same images, bit for bit, and every
  // image is released afterwards.  The stream takes every shape up front and an ImageRef knows its shape only once
  // loaded, so an image that is not loaded yet is first loaded and released once on its own.
  std::vector<std::vector<pano::Descriptor>> detect_lazy(std::vector<pano::ImageRef>& imgs, int window,
                                                         pano_featureset** keep = nullptr) const {
    const int n = (int)imgs.size();
    if (window < 1) window = 1;
    std::vector<int> w(n), h(n);
    for (int k = 0; k < n; ++k) {
      const bool resident = imgs[k].img != nullptr;
      imgs[k].load();
      w[k] = imgs[k].width(); h[k] = imgs[k].height();
      if (!resident) imgs[k].release();
    }
    pano_params p = snapshot_params();
    pano_sift_stream* s = nullptr;
    c_.check(pano_sift_stream_create(c_.get(), n, w.data(), h.data(), &p, &s));
    std::vector<pano::ImageRef*> refs(n);
    for (int k = 0; k < n; ++k) refs[k] = &imgs[k];
    add_windows(refs, window, [&](int first, int count, const void* const* src) {
      c_.check(pano_sift_stream_add(s, first, count, src, PANO_SRC_F32_HOST, 3));
    });
    pano_featureset* fs = nullptr;
    c_.check(pano_sift_stream_finish(s, &fs));
    pano_sift_stream_free(s);
    return unpack_batch(fs, n, keep);
  }
 private:
  std::vector<std::vector<pano::Descriptor>> unpack_batch(pano_featureset* fs, int n, pano_featureset** keep) const {
    std::vector<std::vector<pano::Descriptor>> feats(n);
    for (int k = 0; k < n; ++k) {
      feats[k] = unpack(fs, k, /*real=*/false);
      if (feats[k].empty()) error_exit(ssprintf("Cannot find feature in image %d!\n", k));   // stitcherbase.cc:20-21
    }
    if (keep) *keep = fs; else pano_featureset_free(fs);
    return feats;
  }
  std::vector<pano::Descriptor> unpack(pano_featureset* fs, int k, bool real) const {
    const int m = pano_featureset_count(fs, k);
    if (m < 0) error_exit(pano_last_error(c_.get()));
    std::vector<double> xy(2 * (size_t)m + 2);
    std::vector<float> d(128 * (size_t)m + 1);
    if (m) {
      c_.check(pano_featureset_download(fs, k, real ? nullptr : xy.data(), d.data()));
      if (real) c_.check(pano_featureset_download_real(fs, k, xy.data()));
    }
    std::vector<pano::Descriptor> out(m);
    for (int i = 0; i < m; ++i) {
      out[i].coor = Vec2D(xy[2 * i], xy[2 * i + 1]);
      out[i].descriptor.assign(d.begin() + 128 * (size_t)i, d.begin() + 128 * (size_t)(i + 1));
    }
    return out;
  }
  const Context& c_;
};

// ---- matching: PairWiseMatcher's shape (matcher.hh:40-67) with the exact rule of
// FeatureMatcher::match (matcher.cc:15-71).
class B200PairMatcher {
 public:
  B200PairMatcher(const Context& c, pano_featureset* from_detect) : c_(c), fs_(from_detect), owned_(false) {}
  B200PairMatcher(const Context& c, const std::vector<std::vector<pano::Descriptor>>& feats) : c_(c), owned_(true) {
    const int n = (int)feats.size();
    std::vector<int> cnt(n);
    std::vector<std::vector<float>> buf(n);
    std::vector<const float*> ptr(n);
    for (int i = 0; i < n; ++i) {
      cnt[i] = (int)feats[i].size();
      buf[i].resize(128 * (size_t)cnt[i] + 1);
      for (int k = 0; k < cnt[i]; ++k) memcpy(&buf[i][128 * (size_t)k], feats[i][k].descriptor.data(), 512);
      ptr[i] = buf[i].data();
    }
    c_.check(pano_featureset_upload(c_.get(), n, cnt.data(), ptr.data(), nullptr, &fs_));
  }
  ~B200PairMatcher() { if (owned_) pano_featureset_free(fs_); }
  B200PairMatcher(const B200PairMatcher&) = delete;
  B200PairMatcher& operator=(const B200PairMatcher&) = delete;

  // every task of pairwise_match() / linear_pairwise_match() (stitcher.cc:96-136) in one call
  std::vector<pano::MatchData> match_all(const std::vector<std::pair<int, int>>& tasks) const {
    std::vector<int> ij(2 * tasks.size() + 2);
    for (size_t t = 0; t < tasks.size(); ++t) { ij[2 * t] = tasks[t].first; ij[2 * t + 1] = tasks[t].second; }
    pano_params p = snapshot_params();
    pano_matches m;
    c_.check(pano_match_pairs(c_.get(), fs_, (int)tasks.size(), ij.data(), &p, &m));
    std::vector<pano::MatchData> out(tasks.size());
    for (size_t t = 0; t < tasks.size(); ++t)
      for (int q = 0; q < m.count[t]; ++q)
        out[t].data.emplace_back(m.idx[2 * (m.offset[t] + q)], m.idx[2 * (m.offset[t] + q) + 1]);
    pano_matches_free(&m);
    return out;
  }
  pano::MatchData match(int i, int j) const { return match_all({{i, j}})[0]; }   // = pwmatcher.match(i, j)
 private:
  const Context& c_;
  pano_featureset* fs_ = nullptr;
  bool owned_;
};

// ---- blend: a BlenderBase (blender.hh:14-59).  The std::function the reference passes cannot
// cross a C ABI; it is always the closed form of stitcher_image.cc:142-151, so the caller hands
// over what that lambda closes over (homo_inv) through add_image(), and the projection through
// the constructor.  bands == 0: LinearBlender; bands > 0: MultiBandBlender{bands}.
class B200Blender : public pano::BlenderBase {
 public:
  B200Blender(const Context& c, int bands, int projection, Vec2D resolution, Vec2D proj_min)
      : c_(c), bands_(bands), g_(blend_geom(projection, resolution, proj_min)) {}
  void add_image(const Coor& upper_left, const Coor& bottom_right, pano::ImageRef& img, const pano::Homography& homo_inv) {
    img.load();
    pano_blend_image b;
    b.rgb_hwc = img.img->ptr(); b.w = img.width(); b.h = img.height();
    b.x0 = upper_left.x; b.y0 = upper_left.y; b.x1 = bottom_right.x; b.y1 = bottom_right.y;
    memcpy(b.homo_inv, homo_inv.data, sizeof(double) * 9);
    imgs_.push_back(b);
  }
  // the reference signature: only usable when the closure's parameters were handed over first
  void add_image(const Coor&, const Coor&, pano::ImageRef&, std::function<Vec2D(Coor)>) override {
    error_exit("B200Blender: pass the homography (add_image(ul, br, img, homo_inv)), a closure cannot cross the C ABI");
  }
  Mat32f run() override {
    int ow = 0, oh = 0;
    c_.check(pano_blend_target_size((int)imgs_.size(), imgs_.data(), &ow, &oh));
    Mat32f out(oh, ow, 3);
    pano_params p = snapshot_params();
    c_.check(pano_blend(c_.get(), (int)imgs_.size(), imgs_.data(), &g_, bands_, &p, out.ptr(), ow, oh));
    return out;
  }
 private:
  const Context& c_;
  int bands_;
  pano_blend_geom g_;
  std::vector<pano_blend_image> imgs_;
};

// ---- blend with LAZY_READ's memory contract (blender.cc:38-64, multiband.cc:27,49): run() loads the images
// `window` at a time (add_windows), hands them to a pano_blend_stream and releases them before the next window, so at
// most one window of Mat32f is resident on the host and two on the device.  What B200LazyBlender and
// B200CylinderBlender share; they differ in the stream open() creates.
class B200StreamBlender : public pano::BlenderBase {
 public:
  Mat32f run() override {
    int ow = 0, oh = 0;
    c_.check(pano_blend_target_size((int)imgs_.size(), imgs_.data(), &ow, &oh));
    pano_params p = snapshot_params();
    pano_blend_stream* s = open(p, ow, oh);
    add_windows(refs_, window_, [&](int first, int count, const void* const* src) {
      c_.check(pano_blend_stream_add(s, first, count, src, PANO_SRC_F32_HOST, 3));
    });
    Mat32f out(oh, ow, 3);
    c_.check(pano_blend_stream_finish(s, out.ptr()));
    pano_blend_stream_free(s);
    return out;
  }
 protected:
  B200StreamBlender(const Context& c, int bands, int projection, Vec2D resolution, Vec2D proj_min, int window)
      : c_(c), bands_(bands), window_(window < 1 ? 1 : window), g_(blend_geom(projection, resolution, proj_min)) {}
  // The image blended as a w×h image over [upper_left, bottom_right] with homo_inv, its source read from img
  void add(const Coor& upper_left, const Coor& bottom_right, pano::ImageRef& img, const pano::Homography& homo_inv,
           int w, int h) {
    pano_blend_image b;
    b.rgb_hwc = nullptr; b.w = w; b.h = h;
    b.x0 = upper_left.x; b.y0 = upper_left.y; b.x1 = bottom_right.x; b.y1 = bottom_right.y;
    memcpy(b.homo_inv, homo_inv.data, sizeof(double) * 9);
    imgs_.push_back(b);
    refs_.push_back(&img);
  }
  virtual pano_blend_stream* open(const pano_params& p, int ow, int oh) = 0;

  const Context& c_;
  int bands_, window_;
  pano_blend_geom g_;
  std::vector<pano_blend_image> imgs_;
  std::vector<pano::ImageRef*> refs_;
};

// The output is B200Blender's, bit for bit.  The stream needs every image's shape up front: each ImageRef must have
// been loaded once before run() (as calc_feature() does; ImageRef::release keeps the shape).
class B200LazyBlender : public B200StreamBlender {
 public:
  B200LazyBlender(const Context& c, int bands, int projection, Vec2D resolution, Vec2D proj_min, int window = 1)
      : B200StreamBlender(c, bands, projection, resolution, proj_min, window) {}
  void add_image(const Coor& upper_left, const Coor& bottom_right, pano::ImageRef& img, const pano::Homography& homo_inv) {
    add(upper_left, bottom_right, img, homo_inv, img.width(), img.height());
  }
  void add_image(const Coor&, const Coor&, pano::ImageRef&, std::function<Vec2D(Coor)>) override {
    error_exit("B200LazyBlender: pass the homography (add_image(ul, br, img, homo_inv)), a closure cannot cross the C ABI");
  }
 private:
  pano_blend_stream* open(const pano_params& p, int ow, int oh) override {
    pano_blend_stream* s = nullptr;
    c_.check(pano_blend_stream_create(c_.get(), (int)imgs_.size(), imgs_.data(), &g_, bands_, &p, ow, oh, &s));
    return s;
  }
};

// ---- the two point sets of perspective_correction's getPerspectiveTransform (cylstitcher.cc:139-168): the corners
// of the bundle's first and last images (their half-extents ±0.5 of the WARPED shape first_w×first_h and
// last_w×last_h, through the image's homo, normalised by the identity image's warped shape ref_w×ref_h, projected
// with the bundle's homo2proj, scaled back and moved by -proj_range.min), in the order (-,-) (-,+) of the first and
// (+,-) (+,+) of the last; and the w×h mosaic's corners (0,0), (0,h), (w,0), (w,h) they are stretched to.  The same
// double operations in the same order as the reference, so the points, and the homography solved from them, are
// its bits.
inline void b200_correction_points(const pano::ConnectedImages& bundle, int ref_w, int ref_h, int first_w, int first_h,
                                   int last_w, int last_h, int w, int h, std::vector<Vec2D>* corners,
                                   std::vector<Vec2D>* targets) {
  const auto homo2proj = bundle.get_homo2proj();
  const Vec2D proj_min = bundle.proj_range.min;
  const pano::Homography* homo[2] = {&bundle.component.front().homo, &bundle.component.back().homo};
  const int sw[2] = {first_w, last_w}, sh[2] = {first_h, last_h};
  const double fx[4] = {-0.5, -0.5, 0.5, 0.5}, fy[4] = {-0.5, 0.5, -0.5, 0.5};
  corners->clear();
  for (int q = 0; q < 4; ++q) {
    Vec2D v(fx[q], fy[q]);
    v.x *= sw[q / 2], v.y *= sh[q / 2];
    Vec p = homo[q / 2]->trans(v);
    p.x /= ref_w, p.y /= ref_h;
    Vec2D c = homo2proj(p);
    c.x *= ref_w, c.y *= ref_h;
    corners->push_back(c - proj_min);
  }
  *targets = {Vec2D(0, 0), Vec2D(0, h), Vec2D(w, 0), Vec2D(w, h)};
}

// ---- cylinder mode's warp and blend in one (cylstitcher.cc:24-27, 65-67): CylinderWarper(h_factor).warp of every
// image followed by the flat-projection blend of ConnectedImages::blend, from the UNWARPED images.  run() loads
// them `window` at a time into a cylinder blend stream (pano_blend_stream_create_cyl) and releases them before
// the next window; no warped image is made, on the host or the device.  add_image takes the unwarped ImageRef
// (loaded once before, for its shape) and the range and homo_inv of its warped image; the mosaic is that of
// LinearBlender / MultiBandBlender over the warped images, bit for bit.
class B200CylinderBlender : public B200StreamBlender {
 public:
  B200CylinderBlender(const Context& c, int bands, real_t h_factor, Vec2D resolution, Vec2D proj_min, int window = 1)
      : B200StreamBlender(c, bands, PANO_PROJ_FLAT, resolution, proj_min, window), h_factor_(h_factor) {}
  void add_image(const Coor& upper_left, const Coor& bottom_right, pano::ImageRef& img, const pano::Homography& homo_inv) {
    pano_params p = snapshot_params();
    int w, h;
    double ox, oy;
    c_.check(pano_cyl_warp_shape(img.width(), img.height(), h_factor_, &p, &w, &h, &ox, &oy));
    add(upper_left, bottom_right, img, homo_inv, w, h);
    src_w_.push_back(img.width()); src_h_.push_back(img.height());
  }
  void add_image(const Coor&, const Coor&, pano::ImageRef&, std::function<Vec2D(Coor)>) override {
    error_exit("B200CylinderBlender: pass the homography (add_image(ul, br, img, homo_inv)), a closure cannot cross the C ABI");
  }
  // main.cc:226-233 on CylinderStitcher::build()'s result — crop() when `crop`, then write_rgb(fname) of
  // perspective_correction(run()) — without the f32 mosaic: a cylinder sweep (pano_blend_sweep_create_cyl) of `rows`
  // corrected rows per strip, each blending the band of mosaic rows its correction reads from the unwarped images.
  // corr_inv is perspective_correction's `inv` (cylstitcher.cc:144-168: the four corners of the bundle's first and
  // last images in the identity frame, then getPerspectiveTransform to the w×h rectangle, w×h run()'s shape): a host
  // solve the caller makes, as it makes homo_inv.  An image is loaded (ImageRef::load) for each upload the sweep's
  // plan asks for and released after that strip; keep_bytes bounds the f32 sources kept on the device between
  // strips (SIZE_MAX: no limit).  The file is write_rgb's, byte for byte.  Defined in pano_host_io.hh.
  void write_sweep(const pano::Homography& corr_inv, int rows, size_t keep_bytes, bool crop, const char* fname);
  // write_sweep with perspective_correction's own inv: the bundle CylinderStitcher::build blends (its components in
  // add_image's order, identity_idx, proj_range, the flat projection), the corner points b200_correction_points
  // gives for the warped shapes of add_image's images, and the reference's getPerspectiveTransform
  // (lib/imgproc.cc:251) of them.  The file is write_rgb(crop(CylinderStitcher::build()))'s, byte for byte.
  void write_sweep(const pano::ConnectedImages& bundle, int rows, size_t keep_bytes, bool crop, const char* fname) {
    const int n = (int)imgs_.size();
    m_assert(n > 0 && (int)bundle.component.size() == n && bundle.identity_idx >= 0 && bundle.identity_idx < n);
    int ow = 0, oh = 0;
    c_.check(pano_blend_target_size(n, imgs_.data(), &ow, &oh));
    const pano_blend_image &ref = imgs_[bundle.identity_idx], &first = imgs_.front(), &last = imgs_.back();
    std::vector<Vec2D> corners, targets;
    b200_correction_points(bundle, ref.w, ref.h, first.w, first.h, last.w, last.h, ow, oh, &corners, &targets);
    write_sweep(pano::Homography(pano::getPerspectiveTransform(corners, targets)), rows, keep_bytes, crop, fname);
  }
  // the uploads and loads of the last write_sweep
  long long last_sweep_uploads() const { return last_sweep_uploads_; }
  long last_sweep_loads() const { return last_sweep_loads_; }
 private:
  pano_blend_stream* open(const pano_params& p, int ow, int oh) override {
    pano_blend_stream* s = nullptr;
    c_.check(pano_blend_stream_create_cyl(c_.get(), (int)imgs_.size(), imgs_.data(), src_w_.data(), src_h_.data(),
                                          h_factor_, &g_, bands_, &p, ow, oh, &s));
    return s;
  }
  real_t h_factor_;
  std::vector<int> src_w_, src_h_;
  long long last_sweep_uploads_ = 0;
  long last_sweep_loads_ = 0;
};

// ---- cylinder warp: CylinderWarper(h_factor).warp(mat, kpts) (warp.hh:41-66)
class B200CylinderWarper {
 public:
  B200CylinderWarper(const Context& c, real_t h_factor) : c_(c), h_factor_(h_factor) {}
  void warp(Mat32f& mat, std::vector<Vec2D>& kpts) const {
    pano_params p = snapshot_params();
    int ow, oh;
    double ox, oy;
    c_.check(pano_cyl_warp_shape(mat.width(), mat.height(), h_factor_, &p, &ow, &oh, &ox, &oy));
    Mat32f out(oh, ow, 3);
    std::vector<double> xy(2 * kpts.size() + 2);
    for (size_t i = 0; i < kpts.size(); ++i) { xy[2 * i] = kpts[i].x; xy[2 * i + 1] = kpts[i].y; }
    c_.check(pano_cyl_warp(c_.get(), mat.ptr(), mat.width(), mat.height(), h_factor_, &p, out.ptr(), ow, oh, xy.data(),
                           (int)kpts.size()));
    for (size_t i = 0; i < kpts.size(); ++i) kpts[i] = Vec2D(xy[2 * i], xy[2 * i + 1]);
    mat = out;
  }
 private:
  const Context& c_;
  real_t h_factor_;
};

// ---- the little-planet view: planet() (main.cc:294-331) without its file I/O, so that its body becomes
//   write_rgb(IMGFILE(planet), b200_planet(ctx, read_img(fname)));
inline Mat32f b200_planet(const Context& c, const Mat32f& img) {
  m_assert(img.channels() == 3);
  Mat32f out(PANO_PLANET_SIZE, PANO_PLANET_SIZE, 3);
  c.check(pano_planet(c.get(), img.ptr(), img.width(), img.height(), out.ptr()));
  return out;
}

// ---- Stitcher::build()'s hot path (stitcher.cc:32-64) on the engine: calc_feature ->
// pairwise / linear match -> blend.  The geometry in between (RANSAC, camera estimation,
// bundle adjustment: host code that stays the reference's) is supplied by the caller as the
// per-image ranges and inverse homographies ConnectedImages would hold.
struct StitchGeometry {
  int projection = PANO_PROJ_FLAT;
  Vec2D resolution{1, 1}, proj_min{0, 0};
  std::vector<Coor> upper_left, bottom_right;
  std::vector<pano::Homography> homo_inv;
};

class B200Stitcher {
 public:
  explicit B200Stitcher(const Context& c) : c_(c), det_(c) {}
  // returns the mosaic; feats / matches are left for the host geometry
  Mat32f build(std::vector<pano::ImageRef>& imgs, const StitchGeometry& geo) {
    const int n = (int)imgs.size();
    std::vector<const Mat32f*> mats(n);
    for (int k = 0; k < n; ++k) { imgs[k].load(); mats[k] = imgs[k].img; }
    pano_featureset* fs = nullptr;
    feats = det_.detect_batch(mats, &fs);                                     // calc_feature()
    std::vector<std::pair<int, int>> tasks;
    if (config::ORDERED_INPUT) for (int i = 0; i < n; ++i) tasks.emplace_back(i, (i + 1) % n);       // stitcher.cc:121-122
    else for (int i = 0; i < n; ++i) for (int j = i + 1; j < n; ++j) tasks.emplace_back(i, j);       // stitcher.cc:98-100
    {
      B200PairMatcher pm(c_, fs);
      matches = pm.match_all(tasks);
    }
    pano_featureset_free(fs);
    pairs = tasks;
    B200Blender bl(c_, config::MULTIBAND, geo.projection, geo.resolution, geo.proj_min);              // stitcher_image.cc:132-136
    for (int k = 0; k < n; ++k) bl.add_image(geo.upper_left[k], geo.bottom_right[k], imgs[k], geo.homo_inv[k]);
    return bl.run();
  }
  std::vector<std::vector<pano::Descriptor>> feats;
  std::vector<std::pair<int, int>> pairs;
  std::vector<pano::MatchData> matches;
 private:
  const Context& c_;
  B200SIFTDetector det_;
};

// ---- bundle adjustment: the per-point work of one LM iteration of IncrementalBundleAdjuster::optimize
// (incremental_bundle_adjuster.cc:117-169) on a pano_ba_session.  Constructed where optimize() has
// called update_index_map(), from match_pairs in order; then, per iteration,
//   error(cameras)              replaces calcError(state) (:171-197) incl. update_stats (:199-220)
//   normal_equations(mats, ..)  replaces get_param_update's calcJacobianSymbolic + `J.transpose() * err_vec`
//                               (:233-238); b uses the residuals of the LAST error() call, as the
//                               reference's err_stat.residuals do after a rejected step (:140, :152)
// The damping (:240-248), the solve (:250) and the per-pair 3x3 algebra (the 13 matrices of
// pano_ba_pair, which need the file-local dRdvi) stay in the caller's TU.
class B200BundleAdjusterStep {
 public:
  struct Pair { int from, to; const pano::MatchInfo* m; };   // slots index_map[pair.from], index_map[pair.to]
  struct Stats { double avg, max; };
  B200BundleAdjusterStep(const Context& c, int n_cam, const std::vector<Pair>& pairs) : c_(c), n_cam_(n_cam), pairs_(pairs) {
    std::vector<pano_ba_link> links(pairs.size() + 1);
    std::vector<double> pts;
    int begin = 0;
    for (size_t p = 0; p < pairs.size(); ++p) {
      const int n = (int)pairs[p].m->match.size();
      links[p].from = pairs[p].from; links[p].to = pairs[p].to; links[p].match_begin = begin; links[p].n_match = n;
      for (const auto& q : pairs[p].m->match) {
        pts.push_back(q.first.x); pts.push_back(q.first.y); pts.push_back(q.second.x); pts.push_back(q.second.y);
      }
      begin += n;
    }
    n_res_ = 2 * (size_t)begin;
    c_.check(pano_ba_session_create(c_.get(), n_cam, (int)pairs.size(), links.data(), pts.empty() ? nullptr : pts.data(), &s_));
  }
  ~B200BundleAdjusterStep() { pano_ba_session_free(s_); }
  B200BundleAdjusterStep(const B200BundleAdjusterStep&) = delete;
  B200BundleAdjusterStep& operator=(const B200BundleAdjusterStep&) = delete;

  // calcError(state): `cameras` = state.get_cameras() (slot order).  residuals (optional) as ErrorStats::residuals.
  Stats error(const std::vector<pano::Camera>& cameras, std::vector<double>* residuals = nullptr) {
    std::vector<double> h(9 * pairs_.size() + 1);
    for (size_t p = 0; p < pairs_.size(); ++p) {
      const pano::Camera &c_from = cameras[pairs_[p].from], &c_to = cameras[pairs_[p].to];
      pano::Homography m = (c_from.K() * c_from.R) * (c_to.Rinv() * c_to.K().inverse());   // :182-183
      memcpy(&h[9 * p], m.data, sizeof(double) * 9);
    }
    Stats st;
    if (residuals) residuals->resize(n_res_);
    c_.check(pano_ba_error(s_, (int)pairs_.size(), h.data(), &st.avg, &st.max,
                           residuals && n_res_ ? residuals->data() : nullptr));
    return st;
  }
  // J^T J (undamped, (6 n_cam)^2 row-major) and b = J^T r at the state the 13 matrices per pair
  // (pano_ba_pair.m order, 117 doubles each) were evaluated at.  j_rows (optional): pano_ba_jacobian's layout.
  void normal_equations(const std::vector<double>& mats, std::vector<double>& jtj, std::vector<double>& b,
                        std::vector<double>* j_rows = nullptr) {
    const size_t N = 6 * (size_t)n_cam_;
    jtj.resize(N * N);
    b.resize(N);
    if (j_rows) j_rows->resize(12 * n_res_);
    c_.check(pano_ba_normal_equations(s_, (int)pairs_.size(), mats.data(), jtj.data(), b.data(),
                                      j_rows && n_res_ ? j_rows->data() : nullptr));
  }
 private:
  const Context& c_;
  int n_cam_;
  std::vector<Pair> pairs_;
  size_t n_res_ = 0;
  pano_ba_session* s_ = nullptr;
};

}  // namespace pano_b200
