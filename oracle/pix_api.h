/*
 * pix_api.h — checker API of the reference's decoder and encoder layouts (lib/imgio.cc).  TEST INFRASTRUCTURE ONLY.
 *   - oracle/liboracle_pix.so              orc_ : plain-C restatement (oracle/orc_pix.c)
 *   - oracle/_ref/libopenpano_ref_pix.so   ref_ : the reference's read_img / write_rgb with its own lodepng and CImg
 *                                                 (oracle/refshim/ref_pix.cc)
 * Both are built by oracle/pix_formats.mk.  The interleaved and grey rules stay in oracle_api.h.
 */
#ifndef PIX_API_H
#define PIX_API_H

#ifdef __cplusplus
extern "C" {
#endif

/* read_png (imgio.cc:43-61) on lodepng::decode's h×w×4 buffer: r, g, b each (float)v / 255.0, the fourth
 * byte skipped.  out_hwc: h×w×3 f32.  0, or -1 for a null pointer or w, h < 2 (imgio.cc:89). */
int orc_read_png_rgba(const unsigned char* rgba, int w, int h, float* out_hwc);
/* read_img's spectrum-3 path (imgio.cc:72-83) on CImg<unsigned char>'s planes: sample (x, y, c) at
 * c·w·h + y·w + x, divided by 255 as above. */
int orc_read_img_planar(const unsigned char* planes, int w, int h, float* out_hwc);
/* write_png's buffer (imgio.cc:25-41): h×w×4, (v < 0 ? 1 : v) * 255 truncated, alpha 255. */
int orc_write_png_rgba(const float* mat_hwc, int w, int h, unsigned char* rgba);
/* write_rgb's CImg<unsigned char>(w, h, 1, 3) (imgio.cc:98-113): three h×w planes, the same rule. */
int orc_write_rgb_planar(const float* mat_hwc, int w, int h, unsigned char* planes);

/* The reference's own code, through files in the system temp directory.  Not thread-safe.
 * ref_read_png: lodepng::encode writes `raw` (w×h pixels of lodepng colour type `colortype` — 0 grey, 2 RGB,
 * 3 palette, 4 grey+alpha, 6 RGBA — at `bitdepth` bits, 16-bit samples big-endian as the PNG stores them; a
 * palette image takes its `palette_n` RGBA entries from `palette`) to a .png file; read_img reads it into out_hwc
 * and lodepng::decode (read_png's call) into rgba (h×w×4), the buffer a caller decoding as read_img does holds.
 * 0, or -1 when a step fails. */
int ref_read_png(const unsigned char* raw, int w, int h, int colortype, int bitdepth, const unsigned char* palette,
                 int palette_n, float* out_hwc, unsigned char* rgba);
/* ref_read_cimg: a binary PPM (channels 3) or PGM (channels 1) of the interleaved pixels `pix`; read_img reads
 * it into out_hwc and CImg<unsigned char>(file) into planes (channels · h · w bytes, CImg's layout). */
int ref_read_cimg(const unsigned char* pix, int w, int h, int channels, float* out_hwc, unsigned char* planes);
/* ref_write_png: write_rgb(".png") of the h×w×3 f32 mat, read back with lodepng::decode into rgba (h×w×4). */
int ref_write_png(const float* mat_hwc, int w, int h, unsigned char* rgba);
/* ref_write_cimg: write_rgb(".ppm") of the mat, read back with CImg<unsigned char> into planes (3 · h · w). */
int ref_write_cimg(const float* mat_hwc, int w, int h, unsigned char* planes);

#ifdef __cplusplus
}
#endif
#endif
