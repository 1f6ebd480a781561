// pano_host_io.hh — the drop-in's file boundary in the reference's own codecs (lib/imgio.cc), apart from
// pano_host.hh so that CImg and lodepng only enter the translation units that read or write files.
//   load_pixels       read_img's decode (imgio.cc:67-90) without its f32 conversion: the decoder's own buffer
//                     and format, lodepng's RGBA for a .png, CImg's planes (or grey) otherwise
//   B200PixelBlender  B200LazyBlender's blend (LinearBlender / MultiBandBlender, bit for bit) from such buffers
//   write_mosaic      crop + write_rgb of main.cc:226-234 from a device mosaic: the 8-bit conversion on the
//                     device, lodepng::encode for a .png, CImg::save otherwise
//   B200PixelBlender::write_strips
//                     blend + crop + write_rgb of main.cc:226-234 one strip of canvas rows at a time: no f32
//                     mosaic of the whole canvas, on the host or the device
//   B200PixelBlender::write_sweep
//                     the same from one blend sweep: each source is decoded and uploaded once while later strips
//                     read it (within a byte budget), files decoded on demand
//   B200CylinderBlender::write_sweep
//                     cylinder mode's crop + write_rgb of main.cc:226-233 on CylinderStitcher::build()'s
//                     perspective-corrected mosaic, from one cylinder sweep of the unwarped images
//   b200_planet       planet() of main.cc:294-331 from load_pixels' buffer, left on the device for write_mosaic
// The buffers go to B200SIFTDetector::detect_batch_rgb8, B200PixelBlender or the streams (pano_b200.h) with
// their format as the `channels` argument; no Mat32f of a source is built.  Include after the reference's
// headers are on the include path (-I <reference>/src -isystem <reference>/src/third-party), as pano_host.hh.
#pragma once
#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "pano_host.hh"

#ifndef cimg_display
#define cimg_display 0
#endif
#if !defined(DISABLE_JPEG) && !defined(cimg_use_jpeg)
#define cimg_use_jpeg   // read_img's CImg reads JPEG unless the reference is built with -DDISABLE_JPEG
#endif
// lib/debugutils.hh's one-letter macros (P, PP, PA) collide with CImg's identifiers; imgio.cc includes CImg first
#pragma push_macro("P")
#pragma push_macro("PP")
#pragma push_macro("PA")
#undef P
#undef PP
#undef PA
#include "CImg.h"
#pragma pop_macro("PA")
#pragma pop_macro("PP")
#pragma pop_macro("P")
#include "lodepng/lodepng.h"
#include "lib/utils.hh"

namespace pano_b200 {

// One decoded image as the reference's decoder left it: h×w×4 (PANO_PIX_RGBA), three h×w planes
// (PANO_PIX_RGB_PLANAR) or h×w (PANO_PIX_GREY).
struct Pixels {
  std::vector<unsigned char> data;
  int w = 0, h = 0;
  int format = PANO_PIX_RGB;
  const unsigned char* ptr() const { return data.data(); }
};

// read_img's file handling (imgio.cc:67-90), same checks and messages, without building the Mat32f.
inline Pixels load_pixels(const char* fname) {
  if (!exists_file(fname)) error_exit(ssprintf("File \"%s\" not exists!", fname));
  Pixels px;
  if (endswith(fname, ".png")) {
    unsigned w = 0, h = 0;
    const unsigned error = lodepng::decode(px.data, w, h, fname);
    if (error) error_exit(ssprintf("png encoder error %u: %s", error, lodepng_error_text(error)));
    px.w = (int)w; px.h = (int)h; px.format = PANO_PIX_RGBA;
  } else {
    cimg_library::CImg<unsigned char> img(fname);
    m_assert(img.spectrum() == 3 || img.spectrum() == 1);
    px.w = img.width(); px.h = img.height();
    px.format = img.spectrum() == 3 ? PANO_PIX_RGB_PLANAR : PANO_PIX_GREY;
    px.data.assign(img.data(), img.data() + img.size());
  }
  m_assert(px.h > 1 && px.w > 1);
  return px;
}

// write_rgb's encoder step (imgio.cc:98-113): buf is the cw×ch mosaic in the layout write_mosaic converts to,
// RGBA (alpha 255) for a .png, CImg's planes otherwise.
inline void encode_mosaic(const char* fname, const std::vector<unsigned char>& buf, int cw, int ch) {
  if (endswith(fname, ".png")) {
    const unsigned error = lodepng::encode(fname, buf, (unsigned)cw, (unsigned)ch);
    if (error) error_exit(ssprintf("png encoder error %u: %s", error, lodepng_error_text(error)));
  } else {
    cimg_library::CImg<unsigned char> img(cw, ch, 1, 3);
    memcpy(img.data(), buf.data(), buf.size());
    img.save(fname);
  }
}

// Blends decoded buffers through a pano_blend_stream: the mosaic of LinearBlender / MultiBandBlender (and of
// B200Blender) on read_img's images of the same files, bit for bit.  Consecutive images of one format go in
// windows of up to `window`; the caller keeps the buffers until run() returns.
class B200PixelBlender {
 public:
  B200PixelBlender(const Context& c, int bands, int projection, Vec2D resolution, Vec2D proj_min, int window = 1)
      : c_(c), bands_(bands), window_(window < 1 ? 1 : window) {
    g_.projection = projection; g_.res_x = resolution.x; g_.res_y = resolution.y;
    g_.proj_min_x = proj_min.x; g_.proj_min_y = proj_min.y;
  }
  void add_image(const Coor& upper_left, const Coor& bottom_right, const Pixels& px, const pano::Homography& homo_inv) {
    pano_blend_image b;
    b.rgb_hwc = nullptr; b.w = px.w; b.h = px.h;
    b.x0 = upper_left.x; b.y0 = upper_left.y; b.x1 = bottom_right.x; b.y1 = bottom_right.y;
    memcpy(b.homo_inv, homo_inv.data, sizeof(double) * 9);
    imgs_.push_back(b);
    px_.push_back(&px);
    files_.emplace_back();
  }
  // An image that write_sweep decodes from `fname` (load_pixels) whenever a strip asks for it; w×h is its shape.
  // run() and write_strips take add_image's images only.
  void add_file(const Coor& upper_left, const Coor& bottom_right, const std::string& fname, int w, int h,
                const pano::Homography& homo_inv) {
    pano_blend_image b;
    b.rgb_hwc = nullptr; b.w = w; b.h = h;
    b.x0 = upper_left.x; b.y0 = upper_left.y; b.x1 = bottom_right.x; b.y1 = bottom_right.y;
    memcpy(b.homo_inv, homo_inv.data, sizeof(double) * 9);
    imgs_.push_back(b);
    px_.push_back(nullptr);
    files_.push_back(fname);
  }
  // load_pixels calls write_sweep made so far
  long decodes() const { return decodes_; }
  Mat32f run() {
    const int n = (int)imgs_.size();
    int ow = 0, oh = 0;
    c_.check(pano_blend_target_size(n, imgs_.data(), &ow, &oh));
    pano_params p = snapshot_params();
    pano_blend_stream* s = nullptr;
    c_.check(pano_blend_stream_create(c_.get(), n, imgs_.data(), &g_, bands_, &p, ow, oh, &s));
    for (int k0 = 0; k0 < n;) {
      int k1 = k0 + 1;
      while (k1 < n && k1 - k0 < window_ && px_[k1]->format == px_[k0]->format) ++k1;
      std::vector<const void*> src;
      for (int k = k0; k < k1; ++k) src.push_back(px_[k]->ptr());
      c_.check(pano_blend_stream_add(s, k0, k1 - k0, src.data(), PANO_SRC_RGB8_HOST, px_[k0]->format));
      k0 = k1;
    }
    Mat32f out(oh, ow, 3);
    c_.check(pano_blend_stream_finish(s, out.ptr()));
    pano_blend_stream_free(s);
    return out;
  }

  // main.cc:226-234 on run()'s mosaic — crop() when `crop`, then write_rgb(fname) — without that mosaic: the canvas
  // is blended `rows` rows at a time by row-strip streams (pano_blend_stream_create_rows), each fed only the
  // images that reach its rows (an image that reaches k strips is uploaded k times).  The crop scan carries crop()
  // across the strips, and each strip is converted into an 8-bit canvas that is cropped at the end.  Device memory:
  // one strip's blend state and 12 B per strip pixel, two windows of sources, 3 B per canvas pixel and the
  // encoder's layout of it (4 B per pixel for a .png).  The file is write_rgb's, byte for byte, for canvases up to
  // 80,000 columns wide when `crop`.
  void write_strips(int rows, bool crop, const char* fname) {
    const int n = (int)imgs_.size();
    int ow = 0, oh = 0;
    c_.check(pano_blend_target_size(n, imgs_.data(), &ow, &oh));
    if (rows < 1) rows = 1;
    const bool png = endswith(fname, ".png");
    pano_params p = snapshot_params();
    void *d_strip = nullptr, *d_rgb8 = nullptr, *d_out = nullptr, *d_rect = nullptr;
    int rect[4] = {0, 0, ow, oh};
    c_.check(pano_dev_alloc(c_.get(), (size_t)std::min(rows, oh) * ow * 3 * sizeof(float), &d_strip));
    c_.check(pano_dev_alloc(c_.get(), (size_t)ow * oh * 3, &d_rgb8));
    c_.check(pano_dev_alloc(c_.get(), (size_t)ow * oh * (png ? 4 : 3), &d_out));
    c_.check(pano_dev_alloc(c_.get(), sizeof(rect), &d_rect));
    pano_crop_scan* scan = nullptr;
    if (crop) c_.check(pano_crop_scan_create(c_.get(), ow, oh, &scan));
    std::vector<unsigned char> need(n);
    for (int r0 = 0; r0 < oh; r0 += rows) {
      const int r1 = std::min(oh, r0 + rows);
      pano_blend_stream* s = nullptr;
      c_.check(pano_blend_stream_create_rows(c_.get(), n, imgs_.data(), &g_, bands_, &p, ow, oh, r0, r1, &s));
      c_.check(pano_blend_stream_needs(s, need.data()));
      // windows of up to window_ needed images of one format; the others are passed as null
      for (int k0 = 0; k0 < n;) {
        int fmt = -1, used = 0, k1 = k0;
        std::vector<const void*> src;
        for (; k1 < n; ++k1) {
          if (need[k1]) {
            if (used == window_ || (fmt >= 0 && px_[k1]->format != fmt)) break;
            fmt = px_[k1]->format;
            ++used;
          }
          src.push_back(need[k1] ? px_[k1]->ptr() : nullptr);
        }
        c_.check(pano_blend_stream_add(s, k0, k1 - k0, src.data(), PANO_SRC_RGB8_HOST, fmt < 0 ? PANO_PIX_RGB : fmt));
        k0 = k1;
      }
      c_.check(pano_blend_stream_finish_dev(s, (float*)d_strip));
      pano_blend_stream_free(s);
      if (crop) c_.check(pano_crop_scan_add_dev(scan, (const float*)d_strip, r1 - r0));
      c_.check(pano_mat32f_to_rgb8_dev(c_.get(), (const float*)d_strip, ow, r1 - r0, nullptr,
                                       (unsigned char*)d_rgb8 + (size_t)r0 * ow * 3));
    }
    if (crop) {
      c_.check(pano_crop_scan_rect(scan, rect));
      pano_crop_scan_free(scan);
    }
    c_.check(pano_dev_upload(c_.get(), d_rect, rect, sizeof(rect)));
    c_.check(pano_rgb8_crop_to_pix8_dev(c_.get(), (const unsigned char*)d_rgb8, ow, oh, (const int*)d_rect,
                                        png ? PANO_PIX_RGBA : PANO_PIX_RGB_PLANAR, (unsigned char*)d_out));
    std::vector<unsigned char> buf((size_t)rect[2] * rect[3] * (png ? 4 : 3));
    if (!buf.empty()) c_.check(pano_dev_download(c_.get(), buf.data(), d_out, buf.size()));
    for (void* d : {d_strip, d_rgb8, d_out, d_rect}) c_.check(pano_dev_free(c_.get(), d));
    encode_mosaic(fname, buf, rect[2], rect[3]);
  }

  // write_strips' file from one blend sweep (pano_blend_sweep_*): the strips of `rows` canvas rows run top to
  // bottom, and a source read by several strips stays on the device from the first to the last, as far as
  // keep_bytes (bytes of sources kept between strips; SIZE_MAX: no limit) allows.  A file image is decoded once for
  // each upload the sweep's plan asks for and released after that strip; add_image's buffers are handed over as
  // they are.  Device memory: pano_blend_sweep_create's bound (pano_b200.h) and the encoder's layout of the canvas.
  // The file is write_rgb's, byte for byte, for canvases up to 80,000 columns wide when `crop`.
  void write_sweep(int rows, size_t keep_bytes, bool crop, const char* fname) {
    const int n = (int)imgs_.size();
    int ow = 0, oh = 0;
    c_.check(pano_blend_target_size(n, imgs_.data(), &ow, &oh));
    const bool png = endswith(fname, ".png");
    pano_params p = snapshot_params();
    std::vector<size_t> bytes(n);
    for (int k = 0; k < n; ++k)   // a file's bytes before it is decoded: RGBA for a .png, else 3 planes (grey: 1)
      bytes[k] = px_[k] ? px_[k]->data.size()
                        : (size_t)imgs_[k].w * imgs_[k].h * (endswith(files_[k].c_str(), ".png") ? 4 : 3);
    pano_blend_sweep* s = nullptr;
    c_.check(pano_blend_sweep_create(c_.get(), n, imgs_.data(), &g_, bands_, &p, ow, oh, std::max(rows, 1),
                                     bytes.data(), keep_bytes, crop ? 1 : 0, &s));
    std::vector<unsigned char> want(n);
    std::vector<const void*> src(n);
    std::vector<int> fmt(n);
    std::vector<Pixels> loaded(n);
    int st = 0;
    while ((st = pano_blend_sweep_next(s, want.data())) >= 0) {
      for (int k = 0; k < n; ++k) {
        src[k] = nullptr; fmt[k] = PANO_PIX_RGB;
        if (!want[k]) continue;
        const Pixels* px = px_[k];
        if (!px) {
          loaded[k] = load_pixels(files_[k].c_str());
          ++decodes_;
          m_assert(loaded[k].w == imgs_[k].w && loaded[k].h == imgs_[k].h);
          px = &loaded[k];
        }
        src[k] = px->ptr(); fmt[k] = px->format;
      }
      c_.check(pano_blend_sweep_strip(s, src.data(), fmt.data(), PANO_SRC_RGB8_HOST));
      for (Pixels& px : loaded) px = Pixels();       // pageable: staged by the call
    }
    if (st < -1) c_.check(st);
    void* d_out = nullptr;
    int rect[4] = {0, 0, ow, oh};
    c_.check(pano_dev_alloc(c_.get(), (size_t)ow * oh * (png ? 4 : 3), &d_out));
    c_.check(pano_blend_sweep_finish_dev(s, png ? PANO_PIX_RGBA : PANO_PIX_RGB_PLANAR, (unsigned char*)d_out, rect));
    std::vector<unsigned char> buf((size_t)rect[2] * rect[3] * (png ? 4 : 3));
    if (!buf.empty()) c_.check(pano_dev_download(c_.get(), buf.data(), d_out, buf.size()));
    c_.check(pano_dev_free(c_.get(), d_out));
    long long uploads = 0;
    c_.check(pano_blend_sweep_stats(s, &uploads, nullptr, nullptr));
    last_sweep_uploads_ = uploads;
    pano_blend_sweep_free(s);
    encode_mosaic(fname, buf, rect[2], rect[3]);
  }
  // the hand-overs of the last write_sweep (pano_blend_sweep_stats)
  long long last_sweep_uploads() const { return last_sweep_uploads_; }

 private:
  const Context& c_;
  int bands_, window_;
  pano_blend_geom g_;
  std::vector<pano_blend_image> imgs_;
  std::vector<const Pixels*> px_;
  std::vector<std::string> files_;   // add_file's images (empty for add_image's)
  long decodes_ = 0;
  long long last_sweep_uploads_ = 0;
};

inline void B200CylinderBlender::write_sweep(const pano::Homography& corr_inv, int rows, size_t keep_bytes, bool crop,
                                             const char* fname) {
  const int n = (int)imgs_.size();
  int ow = 0, oh = 0;
  c_.check(pano_blend_target_size(n, imgs_.data(), &ow, &oh));
  const bool png = endswith(fname, ".png");
  pano_params p = snapshot_params();
  std::vector<size_t> bytes(n);
  for (int k = 0; k < n; ++k) bytes[k] = (size_t)src_w_[k] * src_h_[k] * 3 * sizeof(float);
  pano_blend_sweep* s = nullptr;
  c_.check(pano_blend_sweep_create_cyl(c_.get(), n, imgs_.data(), src_w_.data(), src_h_.data(), h_factor_, &g_, bands_,
                                       &p, ow, oh, corr_inv.data, std::max(rows, 1), bytes.data(), keep_bytes,
                                       crop ? 1 : 0, &s));
  std::vector<unsigned char> want(n);
  std::vector<const void*> src(n);
  std::vector<int> fmt(n, 3);
  int st = 0;
  last_sweep_loads_ = 0;
  while ((st = pano_blend_sweep_next(s, want.data())) >= 0) {
    for (int k = 0; k < n; ++k) {
      src[k] = nullptr;
      if (!want[k]) continue;
      refs_[k]->load();
      ++last_sweep_loads_;
      m_assert(refs_[k]->width() == src_w_[k] && refs_[k]->height() == src_h_[k]);
      src[k] = refs_[k]->img->ptr();
    }
    c_.check(pano_blend_sweep_strip(s, src.data(), fmt.data(), PANO_SRC_F32_HOST));
    for (int k = 0; k < n; ++k)   // pageable: staged by the call
      if (want[k]) refs_[k]->release();
  }
  if (st < -1) c_.check(st);
  void* d_out = nullptr;
  int rect[4] = {0, 0, ow, oh};
  c_.check(pano_dev_alloc(c_.get(), (size_t)ow * oh * (png ? 4 : 3), &d_out));
  c_.check(pano_blend_sweep_finish_dev(s, png ? PANO_PIX_RGBA : PANO_PIX_RGB_PLANAR, (unsigned char*)d_out, rect));
  std::vector<unsigned char> buf((size_t)rect[2] * rect[3] * (png ? 4 : 3));
  if (!buf.empty()) c_.check(pano_dev_download(c_.get(), buf.data(), d_out, buf.size()));
  c_.check(pano_dev_free(c_.get(), d_out));
  c_.check(pano_blend_sweep_stats(s, &last_sweep_uploads_, nullptr, nullptr));
  pano_blend_sweep_free(s);
  encode_mosaic(fname, buf, rect[2], rect[3]);
}

// main.cc:226-234 on a device mosaic (h×w×3 f32, Color::NO < 0): crop() when `crop`, then write_rgb(fname).
// The conversion runs on the device into the encoder's layout; the file is what write_rgb writes, byte for byte.
inline void write_mosaic(const Context& c, const float* d_mosaic, int w, int h, bool crop, const char* fname) {
  const bool png = endswith(fname, ".png");
  const int format = png ? PANO_PIX_RGBA : PANO_PIX_RGB_PLANAR;
  void* d_rect = nullptr;
  void* d_out = nullptr;
  int rect[4] = {0, 0, w, h};
  c.check(pano_dev_alloc(c.get(), (size_t)w * h * (png ? 4 : 3), &d_out));
  if (crop) {
    c.check(pano_dev_alloc(c.get(), sizeof(rect), &d_rect));
    c.check(pano_crop_rect_dev(c.get(), d_mosaic, w, h, (int*)d_rect));
  }
  c.check(pano_mat32f_to_pix8_dev(c.get(), d_mosaic, w, h, (const int*)d_rect, format, (unsigned char*)d_out));
  if (crop) c.check(pano_dev_download(c.get(), rect, d_rect, sizeof(rect)));
  const int cw = rect[2], ch = rect[3];
  std::vector<unsigned char> buf((size_t)cw * ch * (png ? 4 : 3));
  c.check(pano_dev_download(c.get(), buf.data(), d_out, buf.size()));
  c.check(pano_dev_free(c.get(), d_out));
  if (d_rect) c.check(pano_dev_free(c.get(), d_rect));
  encode_mosaic(fname, buf, cw, ch);
}

// A device block from pano_dev_alloc, given back to its context with the owner.
struct DevFree {
  const Context* c;
  void operator()(float* d) const { pano_dev_free(c->get(), d); }
};
using DevImage = std::unique_ptr<float, DevFree>;

// planet()'s image (main.cc:294-331) of a decoded file, left on the device (1000×1000×3 f32): the planet of
// read_img's image of the same file, bit for bit, without that image.  The `planet` command becomes
//   write_mosaic(ctx, b200_planet(ctx, load_pixels(fname)).get(), 1000, 1000, false, IMGFILE(planet));
inline DevImage b200_planet(const Context& c, const Pixels& px) {
  void* d_pix = nullptr;
  void* d_out = nullptr;
  c.check(pano_dev_alloc(c.get(), px.data.size(), &d_pix));
  c.check(pano_dev_alloc(c.get(), (size_t)PANO_PLANET_SIZE * PANO_PLANET_SIZE * 3 * sizeof(float), &d_out));
  DevImage out((float*)d_out, DevFree{&c});
  c.check(pano_dev_upload(c.get(), d_pix, px.ptr(), px.data.size()));
  c.check(pano_planet_pix8_dev(c.get(), (const unsigned char*)d_pix, px.format, px.w, px.h, out.get()));
  c.check(pano_dev_free(c.get(), d_pix));
  return out;
}

}  // namespace pano_b200
