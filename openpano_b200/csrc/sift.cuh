// sift.cuh — host-visible structures of the batched SIFT pipeline.
#pragma once
#include "common.cuh"
#include "match_tc.cuh"
#include <memory>

#define SIFT_MAX_OCT 8
#define SIFT_MAX_LEVELS 8        // nscale-1 blurred levels
#define SIFT_MAX_TAPS 32         // kw <= 31
#define SIFT_CAP_DEFAULT 8192    // raw extrema / descriptors per image a batch starts with; the
                                 // capacity is a RUNTIME value that doubles on overflow (the reference's
                                 // vectors are unbounded, extrema.cc:56-57): see featureset_sync_counts
#define SIFT_CAP_MAX (1 << 20)
#define SIFT_MAX_PEAKS 18        // a peak needs two lower neighbours: <= 36/2

struct ImgMeta {
  const void* src;    // input (device): h×w×3 f32, or 8-bit pixels in format `channels`
  int in_w, in_h;
  int w0, h0;         // working size
  float ifx, ify;     // 1/fx (rows), 1/fy (cols) of the working resize
  long long work_off; // working RGB offset in the arena (floats); a trace's arena only holds it
  int channels;       // u8 sources only: the PANO_PIX_* format
};

struct OctMeta {
  int img, oct;
  int w, h;
  int pitch;            // floats per plane row: w rounded up to 32, so rows start on 128-byte lines
                        // (TMA needs 16-byte global strides; warps read / write whole lines)
  float ifx, ify;       // octave resize from the working image (oct > 0)
  long long gauss_off;  // nscale planes: grey + blurred levels (|DoG| is re-formed from them where read)
  long long plane;      // floats per plane = pitch * h
};

struct GaussTable {
  int nlev;
  int rmax;
  int center[SIFT_MAX_LEVELS];
  float taps[SIFT_MAX_LEVELS][SIFT_MAX_TAPS];
};

// All device state of one batched SIFT run.  Kept alive by pano_sift_trace for
// stage inspection; freed right after the run otherwise.
struct SiftWork {
  int n_img = 0, n_oct = 0, n_scale = 0;
  std::vector<ImgMeta> h_img;
  std::vector<OctMeta> h_oct;     // n_img * n_oct
  DevBuf<float> arena;
  size_t arena_floats = 0;
  DevBuf<ImgMeta> d_img;
  DevBuf<OctMeta> d_oct;
  DevBuf<int2> d_tilespan;
  DevBuf<TmaDesc> d_maps;         // [n_img * n_oct]
  int n_tiles = 0;
  int cap = SIFT_CAP_DEFAULT;     // per-image capacity of every candidate / descriptor list below
  // keypoint state, all [n_img * cap] unless noted
  DevBuf<int> cand_count;         // [n_img] + work counters (see sift.cu)
  DevBuf<uint32_t> cand_keys;
  DevBuf<uint32_t> seam_keys;     // [n_img * seam capacity]: tile-perimeter pairs for k_extrema_seams
  DevBuf<uint32_t> sorted_keys;
  DevBuf<pano_sspoint> refined;   // valid flag in .dir < 0 ? no: see kp_valid
  DevBuf<unsigned char> kp_valid;
  DevBuf<int> npeaks;
  DevBuf<float> dirs;             // [n_img * cap * SIFT_MAX_PEAKS]
  int* n_desc = nullptr;          // [n_img]: the featureset's d_count
  DevBuf<int> n_refined;          // [n_img] (for traces)
  DevBuf<int> desc_cand;          // [n_img * cap] candidate index of descriptor
  DevBuf<float> desc_dir;         // [n_img * cap]
};

// What a batch's shape alone decides, kept by the context (pano_ctx::sift_plan) for the next batch of the
// same shape: the work buffers with their arena, the uploaded OctMeta / tile spans / TMA maps (valid
// because the arena stays put), the Gaussian table and the launch sizes.  A repeat batch only uploads its
// ImgMeta (the source pointers) and resets the counters.
struct SiftPlan {
  std::vector<int> key;           // see sift_plan_key: n, cap, every (w, h, source kind), pano_params
  std::unique_ptr<SiftWork> wk;
  size_t bytes = 0;               // device bytes held (counted against the context's cache_limit)
  GaussTable gt;
  bool fast = true;
  size_t seam_cap = 0;
  int max_w0 = 0, max_h0 = 0;
};

struct pano_featureset {
  ~pano_featureset() { ctx_small_pinned_put(ctx, std::move(h_count_pinned)); }
  pano_ctx* ctx = nullptr;
  int n_images = 0;
  DevBuf<float> d_desc;       // rows of 128 f32
  DevBuf<double> d_coor;      // rows of 2 f64 (may be null for uploaded sets)
  double* d_real = nullptr;   // SIFT sets: unscaled real_coor in [0,1), rows of 2 f64 (second half of d_coor's block)
  DevBuf<int> d_count;        // [n_images]
  std::vector<long long> base;  // first row of image i
  std::vector<int> h_count;
  bool counts_on_host = false;
  unsigned counts_token = 0;            // completion marker of the count read-back (ctx_signal)
  bool counts_pending = false;
  PinnedBuf h_count_pinned;            // mapped [2n] ints: the counts, then the candidate counts
  TcOperands tc;              // fp16 tensor-core operands of the descriptors (lazy)
  bool tc_ready = false;
  int error = 0;              // sticky failure of the count read-back (returned by every later use)
  // What a capacity overflow needs to run the batch again with larger lists (SIFT sets only):
  // the sources must stay valid until the counts have been read once (pano_b200.h).
  int cap = 0;                          // per-image row capacity of d_desc / d_coor (0: not a SIFT set)
  std::vector<const void*> src;         // device images
  std::vector<int> src_channels;        // u8 sources: PANO_PIX_* format per image; empty: f32 sources
  std::vector<int> src_w, src_h;
  pano_params src_params;
  DevBuf<unsigned char> owned_block;    // staged upload of the host entry points, freed after the count sync
};

// d_src: h×w×3 f32 device images when channels is null, else 8-bit device images in format channels[i]
int sift_run_batch(pano_ctx* ctx, int n, const void* const* d_src, const int* channels, const int* w, const int* h,
                   const pano_params* p, pano_featureset* fs, std::unique_ptr<SiftWork>* keep, int cap);
int featureset_sync_counts(pano_featureset* fs);
// the per-image list capacity the context's SIFT runs start with (PANO_SIFT_CAP on first use, then grown)
extern "C" int ctx_sift_cap(pano_ctx* ctx);
