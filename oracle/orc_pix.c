/*
 * orc_pix.c — CHECKER (test infrastructure only): plain-C restatement of the layouts the reference's
 * decoders hand read_img and its encoders take from write_rgb (lib/imgio.cc), next to orc_imgio.c's
 * interleaved rules.  Pinned against the reference's own lodepng and CImg by tests/test_oracle_pix_formats.py.
 *
 *   orc_read_png_rgba     read_png's loop over lodepng's RGBA buffer   imgio.cc:43-61
 *   orc_read_img_planar   read_img's spectrum-3 loop over CImg planes  imgio.cc:72-83
 *   orc_write_png_rgba    write_png's buffer                           imgio.cc:25-41
 *   orc_write_rgb_planar  write_rgb's CImg image                       imgio.cc:98-113
 */
#include <stddef.h>
#include "pix_api.h"

/* (float)v / 255.0: the float is promoted, divided in double, rounded to float on the store */
static float div255(unsigned char v) { return (float)((double)(float)v / 255.0); }
static unsigned char to_u8(float v) { return (unsigned char)((v < 0 ? 1 : v) * 255); }

int orc_read_png_rgba(const unsigned char* rgba, int w, int h, float* out_hwc) {
  if (!rgba || !out_hwc || w <= 1 || h <= 1) return -1;
  const size_t n = (size_t)w * h;
  for (size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) out_hwc[i * 3 + c] = div255(rgba[i * 4 + c]);   /* rgba[i * 4 + 3] skipped */
  return 0;
}

int orc_read_img_planar(const unsigned char* planes, int w, int h, float* out_hwc) {
  if (!planes || !out_hwc || w <= 1 || h <= 1) return -1;
  const size_t n = (size_t)w * h;
  for (size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) out_hwc[i * 3 + c] = div255(planes[c * n + i]);
  return 0;
}

int orc_write_png_rgba(const float* mat_hwc, int w, int h, unsigned char* rgba) {
  if (!mat_hwc || !rgba || w <= 0 || h <= 0) return -1;
  const size_t n = (size_t)w * h;
  for (size_t i = 0; i < n; ++i) {
    for (int c = 0; c < 3; ++c) rgba[i * 4 + c] = to_u8(mat_hwc[i * 3 + c]);
    rgba[i * 4 + 3] = 255;
  }
  return 0;
}

int orc_write_rgb_planar(const float* mat_hwc, int w, int h, unsigned char* planes) {
  if (!mat_hwc || !planes || w <= 0 || h <= 0) return -1;
  const size_t n = (size_t)w * h;
  for (size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) planes[c * n + i] = to_u8(mat_hwc[i * 3 + c]);
  return 0;
}
