/*
 * pano_b200.h — C ABI of the B200-native SIFT + match + blend engine.
 *
 * This is the drop-in boundary for the hot path of ppwwyyxx/OpenPano
 * (SURVEY.md §8b).  The reference has no FFI layer: its seams are four C++
 * classes.  Each entry point below names the reference interface it replaces
 * (paths relative to the reference's src/).  Plain pointers and sizes only; no
 * torch / C++ types.  All functions return 0 on success or a negative
 * pano_status; they never call exit().
 *
 * Threading: a pano_ctx owns one CUDA stream, a private stream-ordered memory
 * pool and pinned scratch; calls on one ctx must be serialized by the caller
 * (create one ctx per host thread, or use the *_batch entry points, which is
 * how the reference's `#pragma omp parallel for` over images maps to this
 * engine).  Different contexts may be driven from different host threads at
 * the same time; every entry point makes its context's device current for the
 * calling thread, so a ctx can be used from any thread on a multi-GPU host.
 * Work of different contexts overlaps on the device; order it with pano_event_*.
 */
#ifndef PANO_B200_H
#define PANO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

typedef enum pano_status {
  PANO_OK = 0,
  PANO_ERR_CUDA = -1,        /* a CUDA runtime call failed: pano_last_error() */
  PANO_ERR_INVALID = -2,     /* bad argument (null pointer, non-positive size…) */
  PANO_ERR_CAPACITY = -3,    /* a fixed-capacity device list overflowed */
  PANO_ERR_NO_DEVICE = -4,   /* no CUDA device / extension built without one */
  PANO_ERR_NO_FEATURE = -5   /* reference: error_exit("Cannot find feature…"), stitcherbase.cc:20 */
} pano_status;

/* Limits.  Pair lists have none: matching, RANSAC scoring and bundle adjustment accept any number of
 * pairs.  Image counts are bounded: a featureset, a cylinder-warp or 8-bit conversion batch and a blend
 * take at most PANO_MAX_IMAGES images, a bundle adjustment at most PANO_MAX_IMAGES cameras, and a SIFT
 * batch at most PANO_MAX_SIFT_BATCH images (split larger batches).  Larger calls return
 * PANO_ERR_INVALID and leave the context usable. */
#define PANO_MAX_IMAGES 65535
#define PANO_MAX_SIFT_BATCH 512

/* Handles.  The blend stream, the blend sweep, the SIFT stream and the crop scan keep state between calls and
 * share one contract.  Calls on a handle are calls on its ctx (same threading rule), and the ctx must outlive it.
 * A misuse (each handle lists its own) returns PANO_ERR_INVALID, with the reason in pano_last_error, and launches
 * nothing.  Every failure, a misuse or a CUDA error, is sticky: each later call on the handle returns the same
 * code again and does nothing.  Its free is valid in any state, free(NULL) is a no-op, and the ctx stays
 * usable. */

/* Pixel formats of decoded 8-bit images: the per-image `channels` argument of every 8-bit entry point
 * (pano_sift_detect_batch_rgb8[_dev], pano_sift_stream_add and pano_blend_stream_add with the 8-bit kinds,
 * pano_blend_rgb8_dev, pano_blend_rows_rgb8_dev, pano_cyl_warp_batch_rgb8_dev, pano_planet_pix8[_dev],
 * pano_rgb8_to_mat32f[_batch]_dev)
 * takes one of these.  Batches may mix formats per image; a stream add takes one format for its window.
 * Each reads the f32 image read_img (lib/imgio.cc:67-90) would build from the decoder's buffer, bit for bit:
 *   GREY        h×w u8: CImg's spectrum-1 rule, the value replicated to r, g, b and NOT divided by 255.
 *   RGB         h×w×3 interleaved u8, every sample (float)((double)v / 255.0).
 *   RGBA        h×w×4 interleaved u8, lodepng::decode's output (read_png, imgio.cc:43-61): r, g, b divided
 *               by 255, the fourth byte ignored.  A grey PNG arrives as RGBA with r = g = b and IS divided,
 *               unlike GREY: the same grey pixels give different features in the two formats, as in the
 *               reference.  Device sources must be 4-byte aligned.
 *   RGB_PLANAR  three h×w u8 planes R, G, B: CImg<unsigned char>'s layout (imgio.cc:72-88), divided by 255.
 * Any other value (0, 2, 4 included: the reference refuses a bare 4-channel image) returns
 * PANO_ERR_INVALID. */
#define PANO_PIX_GREY 1
#define PANO_PIX_RGB 3
#define PANO_PIX_RGBA 0x104
#define PANO_PIX_RGB_PLANAR 0x203

/* Snapshot of the reference's mutable config globals (lib/config.hh:24-68,
 * defaults from config.cfg:2-69) that the hot path reads. */
typedef struct pano_params {
  int   sift_working_size;         /* SIFT_WORKING_SIZE 800 */
  int   num_octave;                /* NUM_OCTAVE 4 */
  int   num_scale;                 /* NUM_SCALE 7 */
  float scale_factor;              /* SCALE_FACTOR 1.4142135623 */
  float gauss_sigma;               /* GAUSS_SIGMA 1.4142135623 */
  int   gauss_window_factor;       /* GAUSS_WINDOW_FACTOR 6 */
  float judge_extrema_diff_thres;  /* JUDGE_EXTREMA_DIFF_THRES 2e-3 */
  float contrast_thres;            /* CONTRAST_THRES 4e-2 */
  float pre_color_thres;           /* PRE_COLOR_THRES 5e-2 */
  float edge_ratio;                /* EDGE_RATIO 6 */
  int   calc_offset_depth;         /* CALC_OFFSET_DEPTH 4 */
  float offset_thres;              /* OFFSET_THRES 0.5 */
  float ori_radius;                /* ORI_RADIUS 4.5 */
  int   ori_hist_smooth_count;     /* ORI_HIST_SMOOTH_COUNT 2 */
  int   desc_hist_scale_factor;    /* DESC_HIST_SCALE_FACTOR 3 */
  int   desc_int_factor;           /* DESC_INT_FACTOR 512 */
  float match_reject_next_ratio;   /* MATCH_REJECT_NEXT_RATIO 0.8 */
  float focal_length;              /* FOCAL_LENGTH 37 */
  int   ordered_input;             /* ORDERED_INPUT 0 */
  int   lazy_read;                 /* LAZY_READ 1 */
  int   multiband;                 /* MULTIBAND 0 */
  int   max_output_size;           /* MAX_OUTPUT_SIZE 8000 */
} pano_params;

/* Fills *p with the defaults of the reference's config.cfg. */
void pano_params_default(pano_params* p);

/* One scale-space point: POD image of the reference's SSPoint
 * (feature/feature.hh:33-39). */
typedef struct pano_sspoint {
  int    x, y;            /* Coor coor: integer coordinate in the octave */
  double real_x, real_y;  /* Vec2D real_coor in [0,1) */
  int    pyr_id, scale_id;
  float  dir;
  float  scale_factor;
} pano_sspoint;

/* ---------------------------------------------------------------- context */

typedef struct pano_ctx pano_ctx;

/* Creates an engine context on CUDA device `device`.  `cuda_stream` may be
 * NULL (the ctx creates its own non-blocking stream) or a cudaStream_t cast to
 * void* (e.g. torch.cuda.current_stream().cuda_stream) on which every kernel
 * of this ctx is then launched. */
int  pano_create(pano_ctx** out, int device, void* cuda_stream);
void pano_destroy(pano_ctx* ctx);
/* Device memory: every buffer a ctx needs comes stream-ordered from its own pool, and freed blocks
 * are kept by the ctx for the next request of about the same size (a stitch job asks for the same
 * sizes every time; re-arranging the pool for a 0.9 GB arena was seen to block the host for up to
 * 1.5 s).  The environment variable PANO_CACHE_MB bounds what a ctx keeps (default 32768, 0 = keep
 * nothing); pano_trim hands everything it keeps back to the pool, e.g. before a long idle period. */
int  pano_trim(pano_ctx* ctx);
/* The most device memory the ctx's pool has had in use (cudaMemPoolAttrUsedMemHigh) since creation
 * or the last reset; reset != 0 restarts the mark at what is in use now.  Blocks the ctx keeps for
 * reuse count as in use: set PANO_CACHE_MB=0 or call pano_trim first to see what a call needs. */
int  pano_mem_high_water(pano_ctx* ctx, size_t* bytes, int reset);
/* Message of the last failure on this ctx ("" if none).  ctx may be NULL for
 * the last pano_create failure. */
const char* pano_last_error(const pano_ctx* ctx);
/* Blocks until all work queued on the ctx stream has finished. */
int  pano_sync(pano_ctx* ctx);
/* The stream (cudaStream_t as void*) the ctx launches on. */
void* pano_stream(pano_ctx* ctx);

/* Per-kernel timing (CUDA events on the ctx stream).  When enabled, every
 * kernel launch is bracketed by events; pano_kernel_times reports, per kernel
 * name, the launch count and summed duration since the last reset.  Used by
 * bench.py for the roofline line; adds host overhead, so it is off by default
 * and never on inside a timed end-to-end region. */
int  pano_profile_enable(pano_ctx* ctx, int on);
int  pano_profile_reset(pano_ctx* ctx);
/* names: buffer of cap entries × 64 bytes; returns number of distinct kernels. */
int  pano_profile_read(pano_ctx* ctx, int cap, char* names, int* launches, double* total_ms);
/* Total number of kernels this ctx has launched since creation. */
long long pano_launch_count(const pano_ctx* ctx);
/* Diagnostics: how many descriptor rows the last pano_match_pairs_dev call had to
 * re-scan exactly because the tensor-core nomination was not certain. */
int pano_match_last_exact_rows(const pano_ctx* ctx);
/* Diagnostics: rows of the LARGER sets that the last pano_match_pairs_dev call nominated on request
 * ("columns on demand": on large runs only the smaller set of each pair goes through the first tensor
 * pass; matcher.cc:57-61 walks column j only for rows that passed their own ratio test).  0 when
 * both sets went through the first pass. */
int pano_match_last_nominated_rows(const pano_ctx* ctx);

/* ---------------------------------------------------------------- features
 * Replaces FeatureDetector::detect_feature / SIFTDetector::do_detect_feature
 * (feature/feature.hh:42-57, feature/feature.cc:20-47): working-size resize,
 * ScaleSpace (feature/dog.cc:96-114), DOGSpace (dog.cc:131-143),
 * ExtremaDetector::get_extrema (extrema.cc:36-61), OrientationAssign::work
 * (orientation.cc:22-32), SIFT::get_descriptor (sift.cc:77-85).
 *
 * A pano_featureset holds, per image, the descriptors (n×128 f32, row-major)
 * and coordinates (n×2 f64, image-centred input pixels: (c-0.5)*w) ON THE
 * DEVICE so that matching runs without a host round trip; download copies
 * them out in the reference's Descriptor layout (feature.hh:18-30). */
typedef struct pano_featureset pano_featureset;

/* Host images: n pointers to H×W×3 f32 RGB in [0,1] (Mat32f layout,
 * lib/mat.h:7-60).  Includes H2D of the images.  Pageable buffers are staged and may
 * be reused as soon as the call returns; PINNED buffers (pano_host_alloc /
 * cudaHostAlloc) are read by an asynchronous copy and must stay untouched until the
 * first pano_featureset_count / _download / pano_match_* on the result, or pano_sync.
 *
 * Capacity: per-image keypoint lists start at 8192 entries and are NOT a limit — when
 * an image overflows them (the reference's vectors are unbounded, extrema.cc:56-57) the
 * batch is run again with doubled lists at the first count query, transparently.
 * One parameter limit the reference does not have: descriptor windows of at most 127 pixels
 * radius (sqrt(1/2) * GAUSS_SIGMA * max(1, SCALE_FACTOR) * DESC_HIST_SCALE_FACTOR * 5 <= 127;
 * the defaults give 21) — wider settings return PANO_ERR_INVALID. */
int pano_sift_detect_batch(pano_ctx* ctx, int n, const float* const* rgb_hwc,
                           const int* w, const int* h, const pano_params* p,
                           pano_featureset** out);
/* Same, images already resident in device memory (device pointers).  The images must
 * stay valid until the first count query / download / match on the featureset (they are
 * read again if a keypoint list has to grow). */
int pano_sift_detect_batch_dev(pano_ctx* ctx, int n, const float* const* d_rgb_hwc,
                               const int* w, const int* h, const pano_params* p,
                               pano_featureset** out);
/* Single-image convenience = detect_feature(const Mat32f&). */
int pano_sift_detect(pano_ctx* ctx, const float* rgb_hwc, int w, int h,
                     const pano_params* p, pano_featureset** out);
/* SIFT straight from decoded 8-bit pixels, read_img's input (lib/imgio.cc:72-88): n pointers to
 * h×w×channels[i] interleaved u8, channels 1 or 3 per image.  The featureset equals
 * pano_sift_detect_batch's on read_img's f32 images of the same pixels (channels == 3:
 * (float)((double)v / 255.0); channels == 1: the grey value replicated, not divided), and no f32
 * copy of an image is made: the working-size resize reads the 8-bit taps.
 * _rgb8: host memory, pageable or pinned, with pano_sift_detect_batch's rules (3 B/px cross PCIe).
 * _rgb8_dev: device memory, valid until the first count query / download / match on the featureset.
 * channels[i] may also be PANO_PIX_RGBA or PANO_PIX_RGB_PLANAR (the decoders' own layouts, see PANO_PIX_*;
 * 4 B/px cross PCIe for RGBA).  Null pointers, n <= 0, a value that is no PANO_PIX_* format, a device RGBA
 * image that is not 4-byte aligned or an image under 2×2 return PANO_ERR_INVALID. */
int pano_sift_detect_batch_rgb8(pano_ctx* ctx, int n, const unsigned char* const* pix, const int* w,
                                const int* h, const int* channels, const pano_params* p,
                                pano_featureset** out);
int pano_sift_detect_batch_rgb8_dev(pano_ctx* ctx, int n, const unsigned char* const* d_pix, const int* w,
                                    const int* h, const int* channels, const pano_params* p,
                                    pano_featureset** out);

/* Builds a featureset from host descriptors = PairWiseMatcher ctor
 * (feature/matcher.hh:40-46; matcher.cc:73-88 without the kd-forest).
 * desc[i]: n_kp[i]×128 f32; coor[i] may be NULL. */
int pano_featureset_upload(pano_ctx* ctx, int n_images, const int* n_kp,
                           const float* const* desc, const double* const* coor_xy,
                           pano_featureset** out);
/* The same from DEVICE pointers, queued on the context's stream without a host
 * sync (the sources must stay valid until the stream has passed this call): the
 * receiving side of the multi-GPU descriptor exchange. */
int pano_featureset_import_dev(pano_ctx* ctx, int n_images, const int* n_kp,
                               const float* const* d_desc, const double* const* d_coor_xy,
                               pano_featureset** out);
/* Copies image i's rows device-to-device (the sending side); either may be NULL. */
int pano_featureset_export_dev(pano_featureset* fs, int image, double* d_coor_xy, float* d_desc);
/* All images at once: image 0's rows, then image 1's, ... packed back to back (one launch instead
 * of two copies per image); destinations must be 16-byte aligned. */
int pano_featureset_export_all_dev(pano_featureset* fs, double* d_coor_xy, float* d_desc);
int pano_featureset_num_images(const pano_featureset* fs);
/* Number of descriptors of image i (synchronizes on first use). */
int pano_featureset_count(pano_featureset* fs, int image);
/* Copies image i's results to host: coor_xy (2·n f64) and desc (128·n f32);
 * either may be NULL. */
int pano_featureset_download(pano_featureset* fs, int image, double* coor_xy, float* desc);
/* SIFT sets only: image i's keypoints as SIFTDetector::do_detect_feature returns them
 * (feature/sift.cc:150, Descriptor::coor = SSPoint::real_coor in [0,1)), i.e. BEFORE
 * FeatureDetector::detect_feature scales them to image-centred pixels (feature.cc:20-28).
 * A FeatureDetector subclass returns these and lets the base class do its scaling. */
int pano_featureset_download_real(pano_featureset* fs, int image, double* real_xy);
void pano_featureset_free(pano_featureset* fs);

/* --------------------------------------------------------------- matching
 * Replaces PairWiseMatcher::match(i, j) (feature/matcher.cc:90-135) with the
 * exact rule of FeatureMatcher::match (matcher.cc:15-71), which is the parity
 * contract (SURVEY.md §8c): loop over the smaller set, exact fp32 top-2 with
 * lowest-index ties, two-way ratio test with REJECT_RATIO_SQR = ratio².
 * Output pairs are (idx in image i, idx in image j), ascending index of the
 * smaller set. */
typedef struct pano_matches {
  int  n_pairs;      /* number of image pairs */
  int* count;        /* [n_pairs] matches of pair k */
  int* offset;       /* [n_pairs+1] prefix into idx */
  int* idx;          /* [2*offset[n_pairs]] (first, second) */
} pano_matches;

int  pano_match_pairs(pano_ctx* ctx, pano_featureset* fs, int n_pairs,
                      const int* image_ij /* 2*n_pairs */, const pano_params* p,
                      pano_matches* out);
void pano_matches_free(pano_matches* m);
/* Device-resident variant for the timed-in-HBM bench leg: results stay on the
 * device, only the total match count is returned. */
int  pano_match_pairs_dev(pano_ctx* ctx, pano_featureset* fs, int n_pairs,
                          const int* image_ij, const pano_params* p, int* total_matches);
/* Row-sharded forms (multi-GPU brute-force match, BASELINE config 4): the loop of
 * FeatureMatcher::match over the smaller set (matcher.cc:32: `#pragma omp parallel for` over k)
 * is split into n_shards contiguous shares; this call decides share `shard` of EVERY pair —
 * rows [n_small*shard/n_shards, n_small*(shard+1)/n_shards).  Each share still scans all of the
 * larger set and, for its surviving rows, all of the smaller set (matcher.cc:57-61), so every
 * rank holds both descriptor sets and no collective is needed; the shards' lists, concatenated
 * in shard order, are pano_match_pairs' lists.  (0, 1) is the unsharded call. */
int  pano_match_pairs_shard(pano_ctx* ctx, pano_featureset* fs, int n_pairs, const int* image_ij,
                            const pano_params* p, int shard, int n_shards, pano_matches* out);
int  pano_match_pairs_dev_shard(pano_ctx* ctx, pano_featureset* fs, int n_pairs, const int* image_ij,
                                const pano_params* p, int shard, int n_shards, int* total_matches);
/* FeatureMatcher(f1,f2).match() on two host descriptor arrays
 * (matcher.hh:27-38); pairs_out holds 2*min(n,m) ints. */
int  pano_match_bruteforce(pano_ctx* ctx, const float* desc_a, int n,
                           const float* desc_b, int m, const pano_params* p,
                           int* pairs_out, int* n_pairs_out);

/* ------------------------------------------------- RANSAC inlier scoring
 * Replaces the scoring half of TransformEstimation::get_transform
 * (stitch/transform_estimate.cc:68-85): get_inliers (:132-148) for every hypothesis
 * of every pair, the FIRST hypothesis with the largest inlier count (update_max,
 * lib/utils.hh:58-63) and its inlier flags.  Hypothesis generation (sampling with
 * the caller's seeded generator + the normalised DLT, :89-130) stays on the host. */
typedef struct pano_ransac_pair {
  int n_match;
  const double* kp1_xy;   /* 2*n_match: kp1[match.data[i].first]  (image-centred pixels) */
  const double* kp2_xy;   /* 2*n_match: kp2[match.data[i].second] */
  int n_hyp;
  const double* homos;    /* 9*n_hyp: Homography::data, row-major, image 2 -> image 1 */
  float inlier_thres;     /* ransac_inlier_thres (transform_estimate.cc:47) */
} pano_ransac_pair;
/* best_hyp[k] (-1 when pair k has no hypothesis), best_count[k]; hyp_counts[k] (n_hyp ints)
 * and inlier_flags[k] (n_match bytes) are optional per pair (array or entries may be NULL). */
int pano_ransac_score_pairs(pano_ctx* ctx, int n_pairs, const pano_ransac_pair* pairs, int* best_hyp,
                            int* best_count, int* const* hyp_counts, unsigned char* const* inlier_flags);

/* ------------------------------------- bundle-adjustment Jacobian assembly
 * Replaces the per-point part of IncrementalBundleAdjuster::calcJacobianSymbolic
 * (stitch/incremental_bundle_adjuster.cc:306-383): the two rows of J of every point match
 * (:355-361) and the sums of J^T J (:363-382), bit-identical to the reference's loops.
 * The per-pair 3x3 algebra in front of them (:288-304 and the loop-invariant products inside
 * the loop) is Eigen-backed in the reference (Homography::operator*, inverse,
 * Camera::rotation_to_angle) and stays with the caller, who hands in per pair:
 *   m[0]      Hto_to_from = (fromK * c_from.R) * (toRinv * toKinv)            (:304)
 *   m[1]      c_from.R * toRinv * toKinv                                       (:323)
 *   m[2]      toRinv * toKinv                                                  (:332)
 *   m[3..5]   fromK * dRfromdvi[k]                                             (:333-335)
 *   m[6]      toKinv                                                           (:339,349)
 *   m[7..9]   m * dKdfocal, m * dKdppx, m * dKdppy,  m = fromK * c_from.R * toRinv * toKinv  (:338-345)
 *   m[10..12] (fromK * c_from.R) * dRtodviT[k]                                 (:348-352)
 * row-major Homography::data each. */
typedef struct pano_ba_pair {
  int from, to;         /* camera slots: index_map[pair.from], index_map[pair.to] */
  int match_begin;      /* match_cnt_prefix_sum[pair_idx]: pairs are consecutive, the first starts at 0 */
  int n_match;          /* pair.m.match.size() */
  double m[13][9];
} pano_ba_pair;
/* pts_to: p.first of every match (2 doubles each), all pairs concatenated.
 * j_rows (optional, 24 doubles per match): J(idx, param_idx_from + 0..5), J(idx, param_idx_to + 0..5),
 *   then the same 12 entries of row idx + 1 — every other entry of those rows is zero.
 * jtj: (6 n_cam)^2 doubles, row-major, fully written (JtJ.setZero() + the sums). */
int pano_ba_jacobian(pano_ctx* ctx, int n_cam, int n_pair, const pano_ba_pair* pairs, const double* pts_to,
                     double* j_rows, double* jtj);

/* A bundle-adjustment session: the per-point work of every LM iteration of
 * IncrementalBundleAdjuster::optimize (incremental_bundle_adjuster.cc:117-169) on the device —
 * calcError + ErrorStats::update_stats (:171-220) and get_param_update up to the solve: J, J^T J and
 * b = J^T * err_vec (:230-238).  The match coordinates, J and the residuals of the last
 * pano_ba_error call stay on the context's device between calls; an iteration moves the per-pair
 * matrices up and J^T J, b, avg and max down.  The damping (:240-248) and the solve (:250) stay with
 * the caller.  Calls on a session are calls on its ctx (same threading rule); the ctx must outlive it. */
typedef struct pano_ba_session pano_ba_session;
typedef struct pano_ba_link {
  int from, to, match_begin, n_match;   /* as in pano_ba_pair */
} pano_ba_link;
/* pts: 4 doubles per match, pairs concatenated: p.first.x, p.first.y, p.second.x, p.second.y
 * (MatchInfo::match; first = `to`, second = `from` in calcError, :187). */
int  pano_ba_session_create(pano_ctx* ctx, int n_cam, int n_pair, const pano_ba_link* links, const double* pts,
                            pano_ba_session** out);
void pano_ba_session_free(pano_ba_session* s);
/* calcError(state) + update_stats.  hto_to_from: 9 doubles per pair, (c_from.K() * c_from.R) *
 * (c_to.Rinv() * c_to.K().inverse()) of the state being evaluated (:182-183), row-major.
 * residuals (optional, 2 per match): from.x - transformed.x, from.y - transformed.y in pair then match
 * order.  avg: sqrt of the sequential double sum of the FLOAT squares over residuals.size() (NaN without
 * matches); max: the largest |r|, NaN residuals skipped, 0 if none.  n_pair must be the session's. */
int  pano_ba_error(pano_ba_session* s, int n_pair, const double* hto_to_from, double* avg, double* max,
                   double* residuals);
/* get_param_update (:230-238) up to the damping.  mats: 13*9 doubles per pair, the order of
 * pano_ba_pair.m, of the state J is taken at.  jtj: (6 n_cam)^2 doubles, UNDAMPED, as
 * calcJacobianSymbolic leaves it; b: 6 n_cam doubles, J^T times the residuals of the LAST pano_ba_error
 * call on this session (after a rejected step those belong to the rejected state, as at :140/:152);
 * an entry is NaN when a residual of a pair without its camera is not finite (0 * inf in the reference's
 * dense product), and otherwise the reference's sum, inf included.  j_rows (optional) as in
 * pano_ba_jacobian.  PANO_ERR_INVALID before the first pano_ba_error. */
int  pano_ba_normal_equations(pano_ba_session* s, int n_pair, const double* mats, double* jtj, double* b,
                              double* j_rows);

/* ---------------------------------------------------------- cylinder warp
 * Replaces CylinderWarper(h_factor).warp(Mat32f&, vector<Vec2D>&)
 * (stitch/warp.hh:41-66, warp.cc:25-75). */
/* Output shape and offset for an input of w×h (CylinderProject::project(shape),
 * warp.cc:46-67); host-only arithmetic. */
int pano_cyl_warp_shape(int w, int h, double h_factor, const pano_params* p,
                        int* out_w, int* out_h, double* offset_x, double* offset_y);
/* out_hwc: out_h×out_w×3 f32 (Color::NO = -1 where unmapped); kpts_xy (n_kpts
 * pairs, image-centred) are rewritten in place; may be NULL/0. */
int pano_cyl_warp(pano_ctx* ctx, const float* rgb_hwc, int w, int h, double h_factor,
                  const pano_params* p, float* out_hwc, int out_w, int out_h,
                  double* kpts_xy, int n_kpts);

/* The warp loop of CylinderStitcher::build_warp (cylstitcher.cc:65-67: `REP(k, n) warper.warp(*imgs[k].img,
 * keypoints[k])`) as ONE launch over device-resident images: source and destination stay in HBM (the
 * warped images feed pano_blend_dev), the call is asynchronous on the ctx stream; only the keypoints —
 * a few thousand f64 pairs per image, host arithmetic — are rewritten in place before it returns. */
typedef struct pano_cyl_job {
  const float* d_rgb_hwc;   /* device, h×w×3 f32 */
  int w, h;
  float* d_out_hwc;         /* device, out_h×out_w×3 f32 (sizes from pano_cyl_warp_shape) */
  int out_w, out_h;
  double* kpts_xy;          /* host, n_kpts pairs, image-centred; may be NULL/0 */
  int n_kpts;
} pano_cyl_job;
int pano_cyl_warp_batch_dev(pano_ctx* ctx, int n, const pano_cyl_job* jobs, double h_factor, const pano_params* p);
/* pano_cyl_warp_batch_dev from device 8-bit sources (any PANO_PIX_* format per job, RGBA 4-byte aligned):
 * d_pix[k] is h×w×channels[k] interleaved u8 (channels 1
 * or 3), jobs[k].d_rgb_hwc is ignored and may be NULL.  The warped images equal pano_cyl_warp_batch_dev's on
 * pano_rgb8_to_mat32f_dev's images of the same pixels, bit for bit: every tap is converted as read_img
 * converts it (a grey value is replicated to r, g, b without the division), and no f32 copy of a source is
 * made.  Keypoints are rewritten as pano_cyl_warp_batch_dev rewrites them.  Null pointers, other channel
 * counts, an image under 2×2 or an output size other than pano_cyl_warp_shape's return PANO_ERR_INVALID. */
int pano_cyl_warp_batch_rgb8_dev(pano_ctx* ctx, int n, const pano_cyl_job* jobs, const unsigned char* const* d_pix,
                                 const int* channels, double h_factor, const pano_params* p);

/* ----------------------------------------------------------------- blend
 * Replaces BlenderBase::add_image + run (stitch/blender.hh:14-59) for
 * LinearBlender (blender.cc:24-96) and MultiBandBlender (multiband.cc:19-151).
 * The reference passes an opaque std::function per image; it is always the
 * closed form built at stitcher_image.cc:142-151 (and cylstitcher.cc:176-178),
 * so the ABI takes that form's parameters. */
typedef enum pano_projection { PANO_PROJ_FLAT = 0, PANO_PROJ_CYLINDRICAL = 1, PANO_PROJ_SPHERICAL = 2 } pano_projection;

typedef struct pano_blend_image {
  const float* rgb_hwc;   /* H×W×3 f32, host (pano_blend) or device (pano_blend_dev) */
  int w, h;
  int x0, y0, x1, y1;     /* Range{upper_left, bottom_right}, both inclusive (blender.hh:19-26) */
  double homo_inv[9];     /* ImageComponent::homo_inv (stitcher_image.hh:40-43) */
} pano_blend_image;

typedef struct pano_blend_geom {
  int    projection;             /* pano_projection */
  double res_x, res_y;           /* `resolution` (stitcher_image.cc:119) */
  double proj_min_x, proj_min_y; /* proj_range.min */
} pano_blend_geom;

/* target_size = componentwise max of bottom_right (blender.cc:21, multiband.cc:16). */
int pano_blend_target_size(int n, const pano_blend_image* imgs, int* out_w, int* out_h);
/* bands == 0: LinearBlender::run; bands > 0: MultiBandBlender{bands}::run.
 * out_hwc: out_h×out_w×3 f32, -1 where no image contributes. */
int pano_blend(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g,
               int bands, const pano_params* p, float* out_hwc, int out_w, int out_h);
/* Device-resident variant: imgs[k].rgb_hwc and d_out_hwc are device pointers. */
int pano_blend_dev(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g,
                   int bands, const pano_params* p, float* d_out_hwc, int out_w, int out_h);
/* pano_blend_dev from device 8-bit sources (any PANO_PIX_* format per image, RGBA 4-byte aligned):
 * d_pix[k] is h×w×channels[k] interleaved u8 (channels 1 or
 * 3), imgs[k].rgb_hwc is ignored and may be NULL.  The mosaic is pano_blend_dev's on read_img's f32
 * images of the same pixels, bit for bit: every tap is converted as pano_rgb8_to_mat32f_dev converts
 * it, and no f32 copy of a source is made.  Null pointers, n <= 0, other channel counts or an image
 * under 2×2 return PANO_ERR_INVALID. */
int pano_blend_rgb8_dev(pano_ctx* ctx, int n, const pano_blend_image* imgs, const unsigned char* const* d_pix,
                        const int* channels, const pano_blend_geom* g, int bands, const pano_params* p,
                        float* d_out_hwc, int out_w, int out_h);

/* Rows [row0, row1) of the same mosaic into d_out_rows ((row1-row0)×out_w×3 f32): the
 * strip partition of the canvas across GPUs (every output pixel of
 * LinearBlender::run is independent, blender.cc:37-96, so concatenated strips are
 * bit-identical to pano_blend_dev).  bands > 0 (MultiBandBlender): the strip is computed
 * from every image's ROI clipped to [row0 - H, row1 + H), H = the summed half-widths of
 * the level blurs (6+6+6+9 = 27 rows for 5 bands): a band at level l depends on level 0
 * only within that radius, so concatenated strips are bit-identical as well. */
int pano_blend_rows_dev(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g,
                        int bands, const pano_params* p, float* d_out_rows, int out_w, int out_h,
                        int row0, int row1);
/* The same strip from device 8-bit sources (d_pix / channels as for pano_blend_rgb8_dev): concatenated
 * strips are pano_blend_rgb8_dev's mosaic, bit for bit, linear and multiband.  Only the images that reach
 * the strip are read — for bands > 0 those whose ROI, clipped to [row0 - H, row1 + H), meets the canvas,
 * for bands == 0 those whose ROI meets the strip — so a row-sharded caller needs in device memory only the
 * sources of its strip; the pointers of the others are never dereferenced but must still be non-null. */
int pano_blend_rows_rgb8_dev(pano_ctx* ctx, int n, const pano_blend_image* imgs, const unsigned char* const* d_pix,
                             const int* channels, const pano_blend_geom* g, int bands, const pano_params* p,
                             float* d_out_rows, int out_w, int out_h, int row0, int row1);

/* A blend whose sources arrive in windows: LAZY_READ's memory contract (config.cfg:10-11,
 * blender.cc:38-64, multiband.cc:27,49) on the device.  The mosaic is bit-identical to pano_blend's
 * for every partition of the images into windows and every source kind, 8-bit included: an 8-bit
 * tap is converted exactly as pano_rgb8_to_mat32f_dev converts it.
 *
 * Device memory: besides the canvas state a stream never holds more than two windows of sources.
 * The canvas state, allocated by pano_blend_stream_create, is
 *   bands == 0: 16 B per canvas pixel (the colour sums and the weight plane);
 *   bands > 0:  33 B per ROI pixel (two 4-plane f32 level buffers and a mask; ROI rows padded to 32
 *               pixels) plus 1 B per canvas pixel (the target mask); pano_blend_stream_finish adds the
 *               12 B per canvas pixel of the output;
 * plus the per-image table and, for non-flat projections, 8 B per canvas row and column.  Host
 * sources go through a two-slot device ring, each slot as large as the largest window uploaded
 * through it; device sources are read in place and take no ring memory.
 *
 * A stream is a handle (Handles above).  Its misuses: null pointers, an unknown kind, a value that is no
 * PANO_PIX_* format for 8-bit or other than 3 for f32 sources, a device RGBA source that is not 4-byte aligned,
 * out-of-order, overlapping or excess adds, finish before the last image or twice. */
typedef struct pano_blend_stream pano_blend_stream;
typedef enum pano_src_kind {
  PANO_SRC_F32_DEV = 0,    /* device, h×w×3 f32 (Mat32f layout) */
  PANO_SRC_F32_HOST = 1,   /* host, h×w×3 f32 */
  PANO_SRC_RGB8_DEV = 2,   /* device, 8-bit pixels in the add's PANO_PIX_* format (read_img's input) */
  PANO_SRC_RGB8_HOST = 3   /* host, the same */
} pano_src_kind;
/* imgs / g / bands / p / out_w / out_h as for pano_blend; imgs[k].rgb_hwc is ignored and may be NULL.
 * Builds the projection tables and allocates the canvas state. */
int  pano_blend_stream_create(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g,
                              int bands, const pano_params* p, int out_w, int out_h, pano_blend_stream** out);
/* Adds images [first, first + count): first must be the number of images added so far.  srcs[i] is
 * image first + i in the shape imgs[first + i] gave (w, h; `channels` is one PANO_PIX_* format for the window's
 * 8-bit kinds, 3 for f32).
 * Host sources are uploaded on the stream's own copy stream while the previous window's kernels
 * run.  PAGEABLE host buffers are staged and may be reused as soon as the call returns; PINNED ones
 * (pano_host_alloc / cudaHostAlloc) are read by an asynchronous copy and must stay untouched until
 * the add after the next one, or a finish, has returned.  Device sources are read by kernels queued
 * on the ctx stream: work queued on that stream after this call (the next add, a finish,
 * pano_dev_upload) may overwrite them; other streams wait for a pano_event recorded after it. */
int  pano_blend_stream_add(pano_blend_stream* s, int first, int count, const void* const* srcs, int kind,
                           int channels);
/* Valid once all n images have been added, once per stream.  _dev: d_out_hwc is a device buffer of
 * out_h×out_w×3 f32, written asynchronously on the ctx stream; the host form returns when out_hwc
 * holds the mosaic. */
int  pano_blend_stream_finish_dev(pano_blend_stream* s, float* d_out_hwc);
int  pano_blend_stream_finish(pano_blend_stream* s, float* out_hwc);
void pano_blend_stream_free(pano_blend_stream* s);
/* A blend stream of rows [row0, row1) of the canvas only (0 <= row0 < row1 <= out_h): the strip form of
 * pano_blend_rows_dev with LAZY_READ's windows.  add and free are as above; finish writes
 * (row1 - row0)×out_w×3 f32, and the strips of any partition of the canvas, concatenated, are
 * pano_blend's mosaic bit for bit (every window partition, source kind and PANO_PIX_* format, linear and
 * multiband).  Its canvas state covers the rows only:
 *   bands == 0: 16 B per strip pixel;
 *   bands > 0:  33 B per pixel of each ROI clipped to [row0 - H, row1 + H) (H as for pano_blend_rows_dev)
 *               plus 1 B per strip pixel; finish adds the 12 B per strip pixel of the output.
 * The strip needs only the images pano_blend_rows_rgb8_dev reads for it (see pano_blend_stream_needs).  An
 * add may pass NULL for the others; their sources are never read and take no ring memory, and a window
 * without a needed image queues nothing.  A NULL source for a needed image is a misuse.  A strip that no
 * image reaches finishes as all -1. */
int  pano_blend_stream_create_rows(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g,
                                   int bands, const pano_params* p, int out_w, int out_h, int row0, int row1,
                                   pano_blend_stream** out);
/* A blend stream over cylinder mode's warped images that takes the UNWARPED sources: CylinderStitcher::build's
 * `warper.warp(*imgs[k].img, ...)` (cylstitcher.cc:65-67) and blend of the warped images (:24-27) in one, with
 * LAZY_READ's windows.  imgs[k].w / imgs[k].h are the warped shape and must equal pano_cyl_warp_shape(src_w[k],
 * src_h[k], h_factor, p), else PANO_ERR_INVALID; ranges and homo_inv are those of the warped images.  Each add
 * passes image k's source of src_w[k]×src_h[k] (every kind and PANO_PIX_* format of pano_blend_stream_add);
 * add, finish and free are pano_blend_stream's.  The mosaic is pano_blend_dev's over the images
 * pano_cyl_warp_batch_dev / pano_cyl_warp_batch_rgb8_dev warp from the same sources, bit for bit, for every
 * window partition, linear and multiband: each blend tap computes the warped pixels it reads from the source, with
 * the warp's own operations, so no warped image is ever stored.
 * Device memory: the canvas state and the two windows of (unwarped) sources of pano_blend_stream_create, plus
 * 16 B per warped column per image (the warp's column tables) and a 72 B entry per image.  Keypoints are not
 * touched: pano_cyl_warp_shape's offsets warp them on the host. */
int  pano_blend_stream_create_cyl(pano_ctx* ctx, int n, const pano_blend_image* imgs, const int* src_w,
                                  const int* src_h, double h_factor, const pano_blend_geom* g, int bands,
                                  const pano_params* p, int out_w, int out_h, pano_blend_stream** out);
/* flags[k] (k < n) = 1 if the stream reads image k, else 0.  bands > 0: the images whose ROI, clipped to
 * [row0 - H, row1 + H) on a strip with rows above or below it, keeps a row; bands == 0: the images whose
 * rows [y0, y1] meet [row0, row1).  A stream of the whole canvas needs every image. */
int  pano_blend_stream_needs(const pano_blend_stream* s, unsigned char* flags);

/* A sweep of the canvas's row strips, top to bottom, that hands each source over once while it stays in use:
 * blend, crop() and write_rgb's conversion of pano_blend's mosaic strip by strip (the bytes of
 * pano_rgb8_crop_to_pix8_dev on the canvas the row-strip streams give), with a source kept on the device from
 * the first strip that reads it to the last one, as far as `keep_bytes` allows.
 *
 * The schedule is fixed up front by pano_blend_sweep_plan, which needs no device.  Strip s covers rows
 * [s * strip_rows, min(out_h, (s + 1) * strip_rows)) and reads the images blend_stream_needs reports for a row
 * stream of those rows.  Between strips the sweep keeps at most keep_bytes of sources (src_bytes[k] each) that
 * a later strip reads; when one must make room, the kept source whose next use is farthest away goes (ties: the
 * higher image index).  The sources of the current strip are always on the device.  So keep_bytes = 0 hands
 * over every source each strip reads, strip by strip, and keep_bytes = SIZE_MAX each source that some strip
 * reads exactly once; a source no strip reads is never asked for.
 *
 * pano_blend_sweep_plan: imgs / g / bands / p / out_w / out_h as for pano_blend (g is not read: the read sets
 * do not depend on the projection), strip_rows >= 1, src_bytes[k] > 0.  Every output may be NULL.  With
 * S = ceil(out_h / strip_rows) strips, reads / uploads / kept are S×n flags: strip s reads image k; image k is
 * handed over for strip s; that copy is kept for a later strip.  *uploads and *upload_bytes count the
 * hand-overs, *retained_high is the most bytes kept between two strips.  Bad arguments return
 * PANO_ERR_INVALID. */
int  pano_blend_sweep_plan(int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                           const pano_params* p, int out_w, int out_h, int strip_rows, const size_t* src_bytes,
                           size_t keep_bytes, int* n_strips, unsigned char* reads, unsigned char* uploads,
                           unsigned char* kept, long long* n_uploads, unsigned long long* upload_bytes,
                           unsigned long long* retained_high);
/* The sweep object: create; then, until next returns -1, next and strip; then finish_dev once.
 *
 * Device memory, besides the per-image table and the projection tables (8 B per canvas row and column for
 * non-flat projections, built once):
 *   - one strip's row-stream state (pano_blend_stream_create_rows; the tallest strip's at most), and 12 B per
 *     strip pixel of its f32 rows;
 *   - 3 B per canvas pixel (the 8-bit canvas) plus the output's bytes per canvas pixel (finish_dev's d_out is
 *     the caller's);
 *   - two host sources in a two-slot ring (each slot as large as the largest source uploaded through it): a
 *     host source handed over starts a window of the strip's row stream and is uploaded just before it;
 *   - copies of the kept ones: at most keep_bytes between strips, and during a strip at most keep_bytes plus
 *     the bytes of that strip's sources.
 * Device sources are read in place and take none of the last two.
 *
 * A sweep is a handle (Handles above).  Its misuses: null pointers, bad arguments, a source missing where `want`
 * was set or given where it was not, a source larger than its src_bytes, a strip after the last, finish before
 * the last strip or twice. */
typedef struct pano_blend_sweep pano_blend_sweep;
/* imgs / g / bands / p / out_w / out_h as for pano_blend; strip_rows / src_bytes / keep_bytes as for
 * pano_blend_sweep_plan (src_bytes NULL: w·h·3 per image).  crop != 0: finish_dev crops as crop() does
 * (canvases up to 80,000 columns).  Builds the projection tables and the plan. */
int  pano_blend_sweep_create(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g,
                             int bands, const pano_params* p, int out_w, int out_h, int strip_rows,
                             const size_t* src_bytes, size_t keep_bytes, int crop, pano_blend_sweep** out);
/* The index of the next strip, or -1 once every strip has run.  want (n bytes, may be NULL): 1 for the images
 * the caller must hand to that strip (the plan's uploads), else 0. */
int  pano_blend_sweep_next(pano_blend_sweep* s, unsigned char* want);
/* Runs the next strip.  srcs has n entries, non-null exactly where next's `want` is set; formats[k] is the
 * PANO_PIX_* format of srcs[k] for the 8-bit kinds (3 for f32; formats may be NULL for f32 kinds), and kind
 * one pano_src_kind for every source of the call.  Host sources are uploaded on the sweep's copy stream while
 * the previous strip's kernels run; PAGEABLE buffers are staged and may be reused on return, PINNED ones must
 * stay untouched until the next strip or finish call has returned.  Device sources are read in place, also by
 * the later strips the plan keeps them for: they must stay valid until finish_dev has been queued. */
int  pano_blend_sweep_strip(pano_blend_sweep* s, const void* const* srcs, const int* formats, int kind);
/* Valid once every strip has run, once.  Queues the mosaic's bytes in out_format (PANO_PIX_RGB, _RGBA or
 * _RGB_PLANAR, as pano_rgb8_crop_to_pix8_dev) into d_out (out_w·out_h·(4 for RGBA, else 3) bytes) on the ctx
 * stream and writes the rectangle {x0, y0, width, height} to rect (the whole canvas without crop). */
int  pano_blend_sweep_finish_dev(pano_blend_sweep* s, int out_format, unsigned char* d_out, int rect[4]);
/* What the strips run so far handed over: sources, their src_bytes, and the most bytes kept between two strips
 * (the plan's numbers once every strip has run).  Any output may be NULL. */
int  pano_blend_sweep_stats(const pano_blend_sweep* s, long long* uploads, unsigned long long* upload_bytes,
                            unsigned long long* retained_high);
void pano_blend_sweep_free(pano_blend_sweep* s);

/* Cylinder mode's output end as a sweep: write_rgb(crop(CylinderStitcher::build())) — the blend of the warped
 * images (pano_blend_stream_create_cyl, from the UNWARPED sources) followed by perspective_correction
 * (cylstitcher.cc:139-180) — strip by strip, bit for bit, without the f32 mosaic of the whole canvas.
 * corr_inv is perspective_correction's `inv` (the caller's getPerspectiveTransform of the four corners, a host
 * solve like homo_inv): corrected pixel (j, i) is LinearBlender's one-image blend of the mosaic at
 * inv.trans2d(j, i), with no centre shift and no z test, under LAZY_READ's branch as p selects it.  The corrected
 * canvas has the mosaic's out_w×out_h.
 *
 * Strip s covers corrected rows [s * strip_rows, min(out_h, (s + 1) * strip_rows)) and blends the band of mosaic
 * rows [b0, b1) its bilinear taps can read: where z keeps one sign at the strip's four corner pixels, the rows
 * between floor(min y) and floor(max y) + 1 over those corners, widened by one row on each side and clamped to the
 * mosaic (empty when no tap can land on it); where z changes sign, the whole mosaic.  The band's rows are the
 * mosaic's rows of a row-strip stream, bit for bit, for multiband too.  The images a strip reads are those such a
 * stream of its band reads, and the sources are planned over them as for pano_blend_sweep_plan.
 *
 * pano_blend_sweep_plan_cyl: pano_blend_sweep_plan's arguments and outputs plus corr_inv (required) and band
 * (2 ints per strip, {b0, b1}; may be NULL).  No device needed.
 *
 * pano_blend_sweep_create_cyl: imgs / g / bands / p / out_w / out_h as for pano_blend over the WARPED images;
 * src_w / src_h / h_factor as for pano_blend_stream_create_cyl, which validates them the same way; corr_inv,
 * strip_rows, src_bytes, keep_bytes and crop as above and for pano_blend_sweep_create, with src_bytes NULL meaning
 * src_w·src_h·3 per source.  It returns an ordinary sweep: next / strip / finish_dev / stats / free as above,
 * with the UNWARPED sources handed to strip.
 *
 * Device memory, besides the per-image table and the projection tables:
 *   - the tallest band's row-stream state (pano_blend_stream_create_rows of the band's rows), and 12 B per band
 *     pixel of its f32 rows;
 *   - 12 B per strip pixel of the corrected rows;
 *   - 3 B per canvas pixel (the 8-bit canvas) plus the output's bytes per canvas pixel;
 *   - the two-slot ring and the kept sources, as for pano_blend_sweep_create;
 *   - 16 B per warped column per image (the warps' column tables, built once). */
int  pano_blend_sweep_plan_cyl(int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                               const pano_params* p, int out_w, int out_h, const double corr_inv[9], int strip_rows,
                               const size_t* src_bytes, size_t keep_bytes, int* n_strips, int* band,
                               unsigned char* reads, unsigned char* uploads, unsigned char* kept,
                               long long* n_uploads, unsigned long long* upload_bytes,
                               unsigned long long* retained_high);
int  pano_blend_sweep_create_cyl(pano_ctx* ctx, int n, const pano_blend_image* imgs, const int* src_w,
                                 const int* src_h, double h_factor, const pano_blend_geom* g, int bands,
                                 const pano_params* p, int out_w, int out_h, const double corr_inv[9],
                                 int strip_rows, const size_t* src_bytes, size_t keep_bytes, int crop,
                                 pano_blend_sweep** out);

/* SIFT whose sources arrive in windows: LAZY_READ's feature stage (config.cfg:10-11, calc_feature in
 * stitcherbase.cc:9-27 loads, detects and releases one image at a time) on the device.  For every
 * partition of the images into windows and every source kind, the featureset from pano_sift_stream_finish
 * equals pano_sift_detect_batch's (pano_sift_detect_batch_rgb8's for 8-bit sources) on the same images, bit
 * for bit: counts, coordinates, real coordinates and descriptors, and so the match lists on it.  A stream
 * takes up to PANO_MAX_IMAGES images, PANO_MAX_SIFT_BATCH at most in one add, so one featureset can hold
 * more images than one SIFT batch.
 *
 * Device memory: a stream never holds more than two windows of sources.  Besides them it holds
 *   - the SIFT work buffers and per-image keypoint lists of ONE window, what pano_sift_detect_batch_dev
 *     takes for the images of that window (a list overflow re-runs the window with doubled lists, as the
 *     batch does; the larger lists are the context's starting point from then on);
 *   - the packed rows of finished windows: 544 B per descriptor (128 f32, 2 f64 coordinates, 2 f64 real
 *     coordinates), each image's rows rounded up to 32, and no per-image list capacity;
 *   - in pano_sift_stream_finish only, the featureset's own block of the same packed rows, filled from the
 *     finished windows before they are freed.
 * Host sources go through a two-slot device ring, each slot as large as the largest window uploaded through
 * it; device sources are read in place and take no ring memory.  The work buffers stay with the context for
 * the next window of the same shape, as between batches (PANO_CACHE_MB bounds what it keeps).
 *
 * A stream is a handle (Handles above).  Its misuses are the blend stream's, and more than PANO_MAX_SIFT_BATCH
 * images in one add. */
typedef struct pano_sift_stream pano_sift_stream;
/* w[i] × h[i]: image i's shape (at least 2×2); p: the SIFT parameters of every window. */
int  pano_sift_stream_create(pano_ctx* ctx, int n, const int* w, const int* h, const pano_params* p,
                             pano_sift_stream** out);
/* Adds images [first, first + count): first must be the number of images added so far.  srcs[i] is image
 * first + i, h×w×3 f32 (Mat32f layout) for the f32 kinds and 8-bit pixels in format `channels` for the 8-bit
 * kinds, with pano_src_kind as for pano_blend_stream_add.  The add first queues the upload of host sources on
 * the stream's copy stream, then reads the previous window's counts (waiting for its SIFT, and running it again
 * with doubled lists if it overflowed them), packs its rows and queues this window's SIFT.
 * PAGEABLE host buffers are staged and may be reused as soon as the call returns.  PINNED host buffers
 * (pano_host_alloc / cudaHostAlloc) and device sources are read asynchronously, and read again by a re-run:
 * they must stay valid and untouched until the following add or the finish has returned. */
int  pano_sift_stream_add(pano_sift_stream* s, int first, int count, const void* const* srcs, int kind,
                          int channels);
/* Valid once all n images have been added, once per stream.  Resolves the last window and returns an ordinary
 * featureset (counts already on the host) that outlives the stream; free it with pano_featureset_free. */
int  pano_sift_stream_finish(pano_sift_stream* s, pano_featureset** out);
void pano_sift_stream_free(pano_sift_stream* s);

/* ---------------------------------------------------------- little planet
 * Replaces planet() (main.cc:294-331, the `planet` sub-command) without the file I/O: the
 * stereographic "little planet" view of a mosaic.  The input is any h×w×3 f32 image (the blenders'
 * -1 pixels included); h == 1 or w == 1 is valid and gives an image without any colour, as in the
 * reference.  Output pixel (i, j) is interpolate(mosaic, row, column) (lib/imgproc.cc:135-156) at
 * row = min(h - (hypot(500 - i, 500 - j) / 500) * h, h - 1), column = theta / (2π) * w; pixels at
 * distance 0 or >= 500 from the centre, and Color::NO samples, stay -1.  Bit-identical to the
 * reference: hypot and atan are evaluated once per process on the host with its libm, and each ctx
 * keeps the resulting 16 MB per-pixel table on its device from its first planet call to pano_destroy. */
#define PANO_PLANET_SIZE 1000   /* main.cc:297, OUTSIZE */
/* out_hwc = 1000×1000×3 f32, -1 where nothing maps; host in/out, returns when done. */
int pano_planet(pano_ctx* ctx, const float* rgb_hwc, int w, int h, float* out_hwc);
/* Device in/out (e.g. the mosaic pano_blend_dev leaves on the device), asynchronous on the ctx
 * stream; d_out_hwc holds 1000×1000×3 f32. */
int pano_planet_dev(pano_ctx* ctx, const float* d_rgb_hwc, int w, int h, float* d_out_hwc);
/* The planet straight from a decoded 8-bit image (the `planet` command's read_img input): pix is w×h pixels in
 * `format`, any PANO_PIX_* value (1, 3 or 4 bytes per pixel; planar is three w×h planes).  The output bits equal
 * pano_planet's on read_img's f32 image of the same pixels (pano_rgb8_to_mat32f_dev's image), h == 1 and
 * w == 1 included; no f32 copy of the input is made.  write_rgb's bytes of the result come from
 * pano_mat32f_to_pix8_dev.  Null pointers, w < 1 or h < 1, a value that is no PANO_PIX_* format and a device
 * RGBA source that is not 4-byte aligned return PANO_ERR_INVALID and launch nothing.
 * Host in/out (pix pageable or pinned, uploaded as it is), returns when done: */
int pano_planet_pix8(pano_ctx* ctx, const unsigned char* pix, int format, int w, int h, float* out_hwc);
/* Device in/out, asynchronous on the ctx stream; d_out_hwc holds 1000×1000×3 f32: */
int pano_planet_pix8_dev(pano_ctx* ctx, const unsigned char* d_pix, int format, int w, int h, float* d_out_hwc);

/* --------------------------------------------------------- multi-GPU
 * One process (or host thread) per GPU, one pano_ctx each (SURVEY.md §8e).  The path shards on
 * independent units — images k mod G for SIFT (stitcherbase.cc:14), the pair list of
 * stitcher.cc:98-112 for matching, canvas rows for the blend (blender.cc:79, multiband.cc:75,127)
 * — and has two exchange steps, both NCCL over NVLink on the context's stream:
 *   C1  pano_comm_allgather_features   the descriptor sets every pair task needs
 *   C2  pano_comm_allgather_dev        the row strips of pano_blend_rows_dev -> the mosaic
 * libnccl.so.2 is loaded at run time by the first pano_comm_* call; single-GPU hosts never need it. */
typedef struct pano_comm pano_comm;
/* ncclGetUniqueId: rank 0 calls this and hands the 128 bytes to every rank (file, socket, MPI...). */
int  pano_comm_unique_id(unsigned char id[128]);
/* ncclCommInitRank on ctx's device; collective over all `world` ranks. */
int  pano_comm_create(pano_ctx* ctx, int world, int rank, const unsigned char id[128], pano_comm** out);
/* Wraps a communicator the host already has (ncclComm_t cast to void*); not destroyed by pano_comm_destroy. */
int  pano_comm_adopt(pano_ctx* ctx, void* nccl_comm, int world, int rank, pano_comm** out);
void pano_comm_destroy(pano_comm* c);
int  pano_comm_world(const pano_comm* c);
int  pano_comm_rank(const pano_comm* c);
/* C1: `local` = this rank's images (k = rank, rank + world, ... in ascending k; NULL if it owns none)
 * of n_images_total; *all receives a featureset of all n_images_total images on every rank,
 * bit-identical to detecting them on one GPU.  Device to device, no host staging of descriptors. */
int  pano_comm_allgather_features(pano_comm* c, pano_featureset* local, int n_images_total, pano_featureset** all);
/* C2 (and any other equal-sized exchange): bytes_per_rank from d_send of every rank, concatenated by
 * rank into d_recv (world * bytes_per_rank). */
int  pano_comm_allgather_dev(pano_comm* c, const void* d_send, void* d_recv, size_t bytes_per_rank);

/* ------------------------------------------------ 8-bit image boundary
 * The byte formats either side of the path (SURVEY.md §8f.2-3): decoded 8-bit
 * pixels in, 8-bit mosaic out, so 3 B/px cross PCIe instead of 12.  All
 * pointers are device pointers; work is queued on the context's stream. */
/* read_img's conversion loop (lib/imgio.cc:75-88): channels == 3 -> every
 * sample is (float)((double)v / 255.0); channels == 1 -> the grey value is
 * replicated to R,G,B WITHOUT the division (imgio.cc:84-87).  d_pix is
 * h×w×channels interleaved u8; d_out_hwc is h×w×3 f32.  channels may be any PANO_PIX_* format
 * (RGBA: read_png's rule, the fourth byte ignored; planar: read_img's CImg rule). */
int pano_rgb8_to_mat32f_dev(pano_ctx* ctx, const unsigned char* d_pix, int w, int h, int channels,
                            float* d_out_hwc);
/* The same for n images in one launch (the calc_feature loop reads every image,
 * stitcherbase.cc:14-17).  d_pix[i] must be 4-byte, d_out_hwc[i] 16-byte aligned;
 * the pointer arrays themselves are host arrays of device pointers. */
int pano_rgb8_to_mat32f_batch_dev(pano_ctx* ctx, int n, const unsigned char* const* d_pix, const int* w,
                                  const int* h, const int* channels, float* const* d_out_hwc);
/* crop()'s rectangle (lib/imgproc.cc:200-235): the largest axis-aligned
 * rectangle of pixels whose max(r,g,b) >= 0, first maximum in (line, column)
 * order.  d_rect receives {x0, y0, width, height} (device int[4]). */
int pano_crop_rect_dev(pano_ctx* ctx, const float* d_mat_hwc, int w, int h, int* d_rect);
/* The same rectangle from a mosaic that arrives in row strips, top to bottom, for widths up to 80,000 (the
 * reference's limit on a mosaic's edge; pano_crop_rect_dev takes 40,000).  Between adds the scan keeps
 * O(w) ints and the best rectangle so far on the device.  add: d_strip_hwc is the next `rows` lines of the
 * w-wide f32 mosaic, read by work queued on the ctx stream.  rect: valid once all h lines have been added;
 * waits for the scan and writes {x0, y0, width, height} to the host array, pano_crop_rect_dev's rectangle for
 * every strip partition.  A scan is a handle (Handles above).  Its misuses: bad sizes, more than h lines, a null
 * rect, rect before the last line. */
typedef struct pano_crop_scan pano_crop_scan;
int  pano_crop_scan_create(pano_ctx* ctx, int w, int h, pano_crop_scan** out);
int  pano_crop_scan_add_dev(pano_crop_scan* c, const float* d_strip_hwc, int rows);
int  pano_crop_scan_rect(pano_crop_scan* c, int rect[4]);
void pano_crop_scan_free(pano_crop_scan* c);
/* write_rgb's conversion loop (lib/imgio.cc:98-113) applied to the sub-rectangle
 * d_rect = {x0,y0,cw,ch} (device int[4]; NULL = whole image): every sample is
 * (unsigned char)((v < 0 ? 1 : v) * 255), i.e. Color::NO turns white.  Output
 * is packed ch×cw×3 u8 at d_out (capacity h*w*3). */
int pano_mat32f_to_rgb8_dev(pano_ctx* ctx, const float* d_mat_hwc, int w, int h, const int* d_rect,
                            unsigned char* d_out);
/* The same conversion into the layout an encoder takes: format PANO_PIX_RGB is pano_mat32f_to_rgb8_dev;
 * PANO_PIX_RGBA is write_png's buffer for lodepng (imgio.cc:25-41), ch×cw×4 with alpha 255;
 * PANO_PIX_RGB_PLANAR is write_rgb's CImg<unsigned char>(cw, ch, 1, 3) (imgio.cc:98-113), three ch×cw
 * planes R, G, B.  With a rect the rows or planes are packed to the rect's size.  d_out holds h*w*4 bytes
 * (RGBA) or h*w*3; any other format returns PANO_ERR_INVALID. */
int pano_mat32f_to_pix8_dev(pano_ctx* ctx, const float* d_mat_hwc, int w, int h, const int* d_rect, int format,
                            unsigned char* d_out);
/* pano_mat32f_to_pix8_dev's bytes from the mosaic already converted to 8 bits: d_rgb8 is h×w×3 u8 as
 * pano_mat32f_to_rgb8_dev writes it without a rect (the conversion works sample by sample, so converting
 * before cropping changes no byte), d_rect the crop rectangle (device int[4]; NULL = whole image) and
 * format PANO_PIX_RGB, _RGBA or _RGB_PLANAR as above.  d_out must not overlap d_rgb8. */
int pano_rgb8_crop_to_pix8_dev(pano_ctx* ctx, const unsigned char* d_rgb8, int w, int h, const int* d_rect,
                               int format, unsigned char* d_out);

/* ------------------------------------------------------- device utilities */
int pano_dev_alloc(pano_ctx* ctx, size_t bytes, void** d_ptr);
int pano_dev_free(pano_ctx* ctx, void* d_ptr);
int pano_dev_upload(pano_ctx* ctx, void* d_dst, const void* h_src, size_t bytes);
int pano_dev_download(pano_ctx* ctx, void* h_dst, const void* d_src, size_t bytes);
/* Stream-ordered variants: the host buffer must be pinned and stay valid until
 * pano_sync(); used by the end-to-end path to overlap copies with kernels. */
int pano_dev_upload_async(pano_ctx* ctx, void* d_dst, const void* h_src, size_t bytes);
int pano_dev_download_async(pano_ctx* ctx, void* h_dst, const void* d_src, size_t bytes);

/* Page-locked host memory (cudaHostAlloc) for buffers handed to the async copies
 * and to pano_sift_detect_batch. */
int pano_host_alloc(size_t bytes, void** h_ptr);
int pano_host_free(void* h_ptr);

/* Cross-context ordering.  Several contexts on one device (e.g. an upload ctx, a
 * compute ctx and a download ctx, each with its own stream) can overlap copies
 * with kernels: an event recorded on one ctx's stream can be waited for by
 * another ctx's stream (device-side) or by the host. */
typedef struct pano_event pano_event;
int  pano_event_create(pano_ctx* ctx, pano_event** out);
int  pano_event_record(pano_ctx* ctx, pano_event* ev);        /* on ctx's stream */
int  pano_event_wait(pano_ctx* ctx, pano_event* ev);          /* ctx's stream waits (no host block) */
int  pano_event_sync(pano_event* ev);                         /* host blocks until the event completed */
void pano_event_destroy(pano_event* ev);

/* ------------------------------------------------------ stage inspection
 * Parity-test hooks: run the SIFT chain on ONE host image and keep every
 * intermediate on the device so tests can compare each stage with the oracle
 * (SURVEY.md §4 "per-stage oracle tests"). */
typedef struct pano_sift_trace pano_sift_trace;
int  pano_sift_trace_run(pano_ctx* ctx, const float* rgb_hwc, int w, int h,
                         const pano_params* p, pano_sift_trace** out);
int  pano_sift_trace_working_size(const pano_sift_trace* t, int* w0, int* h0);
int  pano_sift_trace_octave_size(const pano_sift_trace* t, int octave, int* w, int* h);
/* kind: 0 working RGB (3ch, octave ignored), 1 gaussian level i∈[0,nscale),
 * 2 |DoG| level i∈[0,nscale-1) (formed on the host as fabsf(G(i) - G(i+1)): the
 * engine keeps no |DoG| planes), 3 mag level i∈[1,nscale), 4 ort level. */
int  pano_sift_trace_plane(pano_sift_trace* t, int kind, int octave, int level, float* out);
/* stage: 0 raw extrema (x,y,pyr_id,scale_id valid), 1 refined+edge-tested
 * keypoints, 2 oriented keypoints.  Returns count; copies min(count,cap). */
int  pano_sift_trace_points(pano_sift_trace* t, int stage, int cap, pano_sspoint* out);
int  pano_sift_trace_descriptors(pano_sift_trace* t, int cap, double* coor_xy, float* desc);
void pano_sift_trace_free(pano_sift_trace* t);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* PANO_B200_H */
