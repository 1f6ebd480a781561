// planet_pix_test.cc — compiles the drop-in's `planet` command from decoded pixels (load_pixels -> b200_planet ->
// write_mosaic, openpano_b200/host/pano_host_io.hh) against the REFERENCE's headers and runs it next to the
// reference's own command body, write_rgb(IMGFILE(planet), planet(read_img(fname))) (main.cc:294-331): read_img
// and write_rgb from oracle/_ref/libopenpano_ref.so (imgio.cc with its lodepng and CImg), planet() from
// oracle/_ref/libopenpano_ref_planet.so.
//   1. writes PNG files of every colour type with the reference's lodepng (grey, grey+alpha, RGB, RGBA, palette,
//      16-bit RGB and grey), a PPM and a PGM;
//   2. for each, writes the planet to a .png (IMGFILE(planet) of a -DDISABLE_JPEG build) and a .ppm both ways and
//      compares the files byte for byte.
// Built by oracle/planet_pix.mk (needs the reference sources); run by tests/test_gpu_planet_pix8.py on a GPU.
//   planet_pix_test <dir>     dir: where the image files are written
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "pano_host.hh"
#include "pano_host_io.hh"
#include "../../oracle/planet_api.h"

using namespace pano;
using namespace pano_b200;

static int g_fail = 0;
#define CHECK(cond, ...) do { if (!(cond)) { ++g_fail; printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } while (0)

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

static unsigned g_seed = 4242u;
static unsigned rnd() { g_seed = g_seed * 1664525u + 1013904223u; return (g_seed >> 8) & 0xffffff; }

// w×h×3 pixels: a gradient with random discs and a little noise
static std::vector<unsigned char> synth_rgb(int w, int h) {
  std::vector<unsigned char> pix((size_t)w * h * 3);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < 3; ++c)
        pix[((size_t)y * w + x) * 3 + c] = (unsigned char)(30 + (180 * (x + (c + 1) * y)) / (w + 3 * h) + rnd() % 9);
  for (int d = 0; d < (w * h) / 2000; ++d) {
    const int cx = rnd() % w, cy = rnd() % h, r = 2 + rnd() % 16;
    unsigned char col[3] = {(unsigned char)(rnd() & 255), (unsigned char)(rnd() & 255), (unsigned char)(rnd() & 255)};
    for (int y = std::max(0, cy - r); y < std::min(h, cy + r + 1); ++y)
      for (int x = std::max(0, cx - r); x < std::min(w, cx + r + 1); ++x)
        if ((x - cx) * (x - cx) + (y - cy) * (y - cy) <= r * r)
          for (int c = 0; c < 3; ++c) pix[((size_t)y * w + x) * 3 + c] = col[c];
  }
  return pix;
}

// A PNG of lodepng colour type `ct` at `bd` bits from w×h×3 pixels: grey takes channel 0, alpha and the low byte of
// 16-bit samples are random, a palette image indexes a random 256-colour palette by channel 0.
static bool write_png(const std::string& path, const std::vector<unsigned char>& rgb, int w, int h, LodePNGColorType ct,
                      unsigned bd) {
  lodepng::State st;
  st.encoder.auto_convert = 0;
  st.info_raw.colortype = st.info_png.color.colortype = ct;
  st.info_raw.bitdepth = st.info_png.color.bitdepth = bd;
  if (ct == LCT_PALETTE) {
    for (int k = 0; k < 256; ++k) {
      const unsigned char r = rnd() & 255, g = rnd() & 255, b = rnd() & 255;
      lodepng_palette_add(&st.info_png.color, r, g, b, 255);
      lodepng_palette_add(&st.info_raw, r, g, b, 255);
    }
  }
  std::vector<unsigned char> raw;
  for (size_t i = 0; i < (size_t)w * h; ++i) {
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

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: planet_pix_test <dir>\n"); return 2; }
  const std::string dir = argv[1];
  Context ctx(0);
  struct File { const char* name; int ct, bd, w, h; };   // ct < 0: PNM of -ct channels
  const File files[] = {{"grey.png", LCT_GREY, 8, 720, 160},    {"grey_alpha.png", LCT_GREY_ALPHA, 8, 640, 200},
                        {"rgb.png", LCT_RGB, 8, 900, 170},      {"rgba.png", LCT_RGBA, 8, 801, 143},
                        {"palette.png", LCT_PALETTE, 8, 500, 120}, {"rgb16.png", LCT_RGB, 16, 600, 150},
                        {"grey16.png", LCT_GREY, 16, 333, 111}, {"rgb.ppm", -3, 8, 1200, 240},
                        {"grey.pgm", -1, 8, 777, 180}};
  for (const File& fl : files) {
    const std::string path = dir + "/" + fl.name;
    const std::vector<unsigned char> rgb = synth_rgb(fl.w, fl.h);
    const bool ok = fl.ct >= 0 ? write_png(path, rgb, fl.w, fl.h, (LodePNGColorType)fl.ct, (unsigned)fl.bd)
                               : write_pnm(path, rgb, fl.w, fl.h, -fl.ct);
    if (!ok) { printf("FAIL: cannot write %s\n", path.c_str()); return 2; }

    // the reference: planet(read_img(fname)), then write_rgb
    const Mat32f img = read_img(path.c_str());
    Mat32f planet(PANO_PLANET_SIZE, PANO_PLANET_SIZE, 3);
    if (ref_planet(img.ptr(), img.width(), img.height(), planet.ptr()) != 0) { printf("ref_planet refused %s\n", fl.name); return 2; }
    const Pixels px = load_pixels(path.c_str());
    for (const char* ext : {".png", ".ppm"}) {
      const std::string ref_path = path + ".ref_planet" + ext, mine_path = path + ".b200_planet" + ext;
      write_rgb(ref_path.c_str(), planet);
      // the drop-in: no f32 image on the host
      write_mosaic(ctx, b200_planet(ctx, px).get(), PANO_PLANET_SIZE, PANO_PLANET_SIZE, false, mine_path.c_str());
      const std::vector<unsigned char> a = file_bytes(ref_path), b = file_bytes(mine_path);
      const bool same = !a.empty() && a == b;
      CHECK(same, "%s -> planet%s: %zu reference bytes, %zu from the drop-in", fl.name, ext, a.size(), b.size());
      if (same) printf("planet %s (%dx%d, format %#x) -> %s: %zu file bytes identical\n", fl.name, fl.w, fl.h, px.format,
                       ext, a.size());
    }
  }
  printf(g_fail ? "PLANET PIX TEST FAILED (%d)\n" : "PLANET PIX TEST OK\n", g_fail);
  return g_fail ? 1 : 0;
}
