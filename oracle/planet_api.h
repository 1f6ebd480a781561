/*
 * planet_api.h — checker API of the little-planet view (main.cc:294-331).  TEST INFRASTRUCTURE ONLY.
 *   - oracle/liboracle_planet.so              orc_ : plain-C restatement (oracle/orc_planet.c)
 *   - oracle/_ref/libopenpano_ref_planet.so   ref_ : the reference's own planet() (oracle/refshim/ref_planet.cc)
 * Both are built by oracle/planet.mk.
 */
#ifndef PLANET_API_H
#define PLANET_API_H

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_PLANET_SIZE 1000   /* main.cc:297 OUTSIZE */

/* planet() on an h×w×3 f32 image (rgb_hwc) without the file I/O: out_hwc receives the 1000×1000×3 f32
 * image planet() hands to write_rgb.  0 on success, -1 for w < 1 or h < 1. */
int orc_planet(const float* rgb_hwc, int w, int h, float* out_hwc);
/* The same through the reference's own planet(): read_img / write_rgb replaced by an in-memory
 * hand-over.  Not thread-safe (the hand-over goes through file-scope variables). */
int ref_planet(const float* rgb_hwc, int w, int h, float* out_hwc);

#ifdef __cplusplus
}
#endif
#endif
