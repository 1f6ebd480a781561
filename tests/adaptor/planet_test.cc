// planet_test.cc — compiles the drop-in's little-planet view (b200_planet, openpano_b200/host/pano_host.hh)
// against the REFERENCE's headers and runs it next to the reference's own planet() (main.cc:294-331, from
// oracle/_ref/libopenpano_ref_planet.so, which hands the image over in memory instead of through files).
// Every output float must be bit-identical.  Each image is run twice on one context: the second call uses
// the per-pixel table the first one uploaded.
// Built by oracle/planet.mk (needs the reference sources); run by tests/test_gpu_planet.py on a GPU.
//   planet_test <img.bin>...   img.bin: int32 w, h; float32 pixels[h][w][3]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "pano_host.hh"
#include "../../oracle/planet_api.h"

using namespace pano_b200;

static int g_fail = 0;
#define CHECK(cond, ...) do { if (!(cond)) { ++g_fail; printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } while (0)

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: planet_test img.bin...\n"); return 2; }
  Context ctx(0);
  const size_t n_out = (size_t)PANO_PLANET_SIZE * PANO_PLANET_SIZE * 3;
  for (int a = 1; a < argc; ++a) {
    FILE* f = fopen(argv[a], "rb");
    if (!f) { perror(argv[a]); return 2; }
    int hdr[2];
    if (fread(hdr, 4, 2, f) != 2) return 2;
    const int w = hdr[0], h = hdr[1];
    Mat32f img(h, w, 3);
    if (fread(img.ptr(), 4, (size_t)w * h * 3, f) != (size_t)w * h * 3) return 2;
    fclose(f);

    std::vector<float> want(n_out);
    if (ref_planet(img.ptr(), w, h, want.data()) != 0) { printf("ref_planet refused %dx%d\n", w, h); return 2; }
    size_t coloured = 0;
    for (size_t k = 0; k < n_out; k += 3) coloured += want[k] >= 0;
    for (int run = 0; run < 2; ++run) {
      Mat32f got = b200_planet(ctx, img);
      CHECK(got.width() == PANO_PLANET_SIZE && got.height() == PANO_PLANET_SIZE && got.channels() == 3,
            "%dx%d: output is %dx%dx%d", w, h, got.width(), got.height(), got.channels());
      CHECK(memcmp(got.ptr(), want.data(), n_out * sizeof(float)) == 0, "%dx%d run %d: planet differs", w, h, run);
    }
    printf("planet %dx%d: %zu pixels with colour, identical\n", w, h, coloured);
  }
  printf(g_fail ? "PLANET TEST FAILED (%d)\n" : "PLANET TEST OK\n", g_fail);
  return g_fail ? 1 : 0;
}
