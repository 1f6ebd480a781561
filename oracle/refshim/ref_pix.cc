// ref_pix.cc — drives the REFERENCE's read_img / write_rgb (lib/imgio.cc) with its own lodepng and CImg
// (compiled unmodified into libopenpano_ref.so and included from the reference tree) and hands back the
// buffers those decoders produce, so the layouts the engine takes and returns are pinned against the
// reference's own code.  TEST INFRASTRUCTURE ONLY; contains no algorithm.  Built by oracle/pix_formats.mk.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <unistd.h>

#define cimg_display 0
#include "CImg.h"
#include "lib/mat.h"
#include "lib/imgproc.hh"
#include "lodepng/lodepng.h"
#include "../pix_api.h"

using namespace pano;

namespace {

std::string temp_name(const char* suffix) {
  const char* dir = getenv("TMPDIR");
  std::string pat = std::string(dir && *dir ? dir : "/tmp") + "/pano_ref_pix_XXXXXX" + suffix;
  std::vector<char> buf(pat.begin(), pat.end());
  buf.push_back(0);
  int fd = mkstemps(buf.data(), (int)strlen(suffix));
  if (fd >= 0) close(fd);
  return buf.data();
}

bool copy_mat(const Mat32f& m, int w, int h, float* out) {
  if (m.width() != w || m.height() != h || m.channels() != 3) return false;
  memcpy(out, m.ptr(), sizeof(float) * 3 * (size_t)w * h);
  return true;
}

}  // namespace

extern "C" {

int ref_read_png(const unsigned char* raw, int w, int h, int colortype, int bitdepth, const unsigned char* palette,
                 int palette_n, float* out_hwc, unsigned char* rgba) {
  lodepng::State st;
  st.encoder.auto_convert = 0;   // keep the colour type asked for
  st.info_raw.colortype = st.info_png.color.colortype = (LodePNGColorType)colortype;
  st.info_raw.bitdepth = st.info_png.color.bitdepth = (unsigned)bitdepth;
  for (int k = 0; k < palette_n; ++k) {
    const unsigned char* e = palette + 4 * k;
    lodepng_palette_add(&st.info_png.color, e[0], e[1], e[2], e[3]);
    lodepng_palette_add(&st.info_raw, e[0], e[1], e[2], e[3]);
  }
  std::vector<unsigned char> png;
  if (lodepng::encode(png, raw, (unsigned)w, (unsigned)h, st)) return -1;
  const std::string fname = temp_name(".png");
  if (lodepng::save_file(png, fname)) { unlink(fname.c_str()); return -1; }
  const Mat32f m = read_img(fname.c_str());
  std::vector<unsigned char> dec;
  unsigned dw = 0, dh = 0;
  const unsigned err = lodepng::decode(dec, dw, dh, fname);
  unlink(fname.c_str());
  if (err || (int)dw != w || (int)dh != h || !copy_mat(m, w, h, out_hwc)) return -1;
  memcpy(rgba, dec.data(), dec.size());
  return 0;
}

int ref_read_cimg(const unsigned char* pix, int w, int h, int channels, float* out_hwc, unsigned char* planes) {
  if (channels != 1 && channels != 3) return -1;
  const std::string fname = temp_name(channels == 3 ? ".ppm" : ".pgm");
  FILE* f = fopen(fname.c_str(), "wb");
  if (!f) return -1;
  fprintf(f, "P%d\n%d %d\n255\n", channels == 3 ? 6 : 5, w, h);
  fwrite(pix, 1, (size_t)w * h * channels, f);
  fclose(f);
  const Mat32f m = read_img(fname.c_str());
  cimg_library::CImg<unsigned char> img(fname.c_str());
  unlink(fname.c_str());
  if (img.width() != w || img.height() != h || img.spectrum() != channels || !copy_mat(m, w, h, out_hwc)) return -1;
  memcpy(planes, img.data(), (size_t)w * h * channels);
  return 0;
}

int ref_write_png(const float* mat_hwc, int w, int h, unsigned char* rgba) {
  Mat32f m(h, w, 3);
  memcpy(m.ptr(), mat_hwc, sizeof(float) * 3 * (size_t)w * h);
  const std::string fname = temp_name(".png");
  write_rgb(fname.c_str(), m);
  std::vector<unsigned char> dec;
  unsigned dw = 0, dh = 0;
  const unsigned err = lodepng::decode(dec, dw, dh, fname);
  unlink(fname.c_str());
  if (err || (int)dw != w || (int)dh != h) return -1;
  memcpy(rgba, dec.data(), dec.size());
  return 0;
}

int ref_write_cimg(const float* mat_hwc, int w, int h, unsigned char* planes) {
  Mat32f m(h, w, 3);
  memcpy(m.ptr(), mat_hwc, sizeof(float) * 3 * (size_t)w * h);
  const std::string fname = temp_name(".ppm");
  write_rgb(fname.c_str(), m);
  cimg_library::CImg<unsigned char> img(fname.c_str());
  unlink(fname.c_str());
  if (img.width() != w || img.height() != h || img.spectrum() != 3) return -1;
  memcpy(planes, img.data(), (size_t)w * h * 3);
  return 0;
}

}  // extern "C"
