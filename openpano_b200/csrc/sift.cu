// sift.cu — batched SIFT on sm_90a: every octave's grey plane in one pass, fused
// 6-sigma separable blur + |DoG| + extremum test, seam scan + ordered compaction,
// sub-pixel refinement, orientation assignment and 128-D RootSIFT descriptors.
//
// Replaces (reference paths relative to src/): feature/feature.cc:20-47,
// feature/dog.cc:42-143, feature/gaussian.hh:29-90, feature/extrema.cc:36-216,
// feature/orientation.cc:22-100, feature/sift.cc:15-152, lib/imgproc.cc:22-80,
// :237-249.  One launch per stage covers every image and octave of the batch.
#include "sift.cuh"
#include "desc_interval.h"
#include <math.h>
#include <string.h>
#include <algorithm>
#include <map>
#include <mutex>
#include <cuda.h>   // CUtensorMap types only: the encoder is looked up at run time

// ============================================================ K1 pyramid grey
// lib/imgproc.cc:22-80 resize_bilinear; the reference's per-row/col tables are
// recomputed per thread with the same float expressions.
__device__ __forceinline__ void bilinear_coef(int d, float inv, int src_n, int* s, float* frac) {
  float r = ((float)d + 0.5f) * inv - 0.5f;
  int si = (int)floorf(r);
  r -= (float)si;
  if (si < 0) { si = 0; r = 0.f; }
  else if (si + 1 >= src_n) { si = src_n - 2; r = 1.f; }
  *s = si; *frac = r;
}

// The smallest d in [0, dst_n) whose lower tap (bilinear_coef(d, inv, src_n)) is >= t, dst_n if
// there is none.  The tap does not decrease as d grows (floor, monotone float rounding and both
// clamps keep order), so a few steps either way correct the estimate.
__device__ __forceinline__ int first_tap_at_least(int t, float inv, int src_n, int dst_n) {
  auto tap = [&](int d) { int s; float f; bilinear_coef(d, inv, src_n, &s, &f); return s; };
  int d = (int)fminf(fmaxf(((float)t + 0.5f) / inv - 0.5f, 0.f), (float)dst_n);
  while (d > 0 && tap(d - 1) >= t) --d;
  while (d < dst_n && tap(d) < t) ++d;
  return d;
}

#define PG_TW 64          // working pixels of one k_pyramid_grey tile: columns
#define PG_TH 32          //                                             rows
#define PG_THREADS 256    // at least 256: build_rgb8_lut

// Every octave's grey plane of one tile of the working image (feature/feature.cc:33-35 working
// resize, feature/dog.cc:96-114 octaves resized from the WORKING image, lib/imgproc.cc:237-249
// rgb2grey), without the working RGB image in HBM.  grid = (tile columns, tile rows, image).
//  1. The working RGB of the tile plus one halo row and column (clamped to h0-1 / w0-1) goes to
//     shared memory as three planes; the tile's own pixels also give octave 0's grey.
//  2. An octave pixel belongs to the tile that holds its lower tap, bilinear_coef(d, ifx, h0) for
//     rows and likewise for columns.  That rule depends on d alone, so every octave pixel is
//     written once, and a tile owns a contiguous range of rows and of columns
//     (first_tap_at_least).  Its upper tap, at most h0-1 / w0-1, is the halo at the latest.
// Every stored value comes from the same float operations on the same operands as the reference's
// resize and rgb2grey (no FMA contraction, --fmad=false), so every plane is bit-identical to them.
// Src = SrcRgb8 / SrcPix8: every tap is the f32 value read_img would have stored (common.cuh), so the
// bilinear sample of those taps is the sample of read_img's image.
// work: null, or the arena when a trace keeps the working RGB image (at im.work_off).
template <class Src>
__global__ void __launch_bounds__(PG_THREADS) k_pyramid_grey(const ImgMeta* __restrict__ imgs,
                                                             const OctMeta* __restrict__ octs, int n_oct,
                                                             float* __restrict__ arena, float* work) {
  constexpr int SW = PG_TW + 1, SP = SW * (PG_TH + 1);   // planar: the octave taps of a warp stay a word apart
  __shared__ float tile[3 * SP];
  __shared__ float lut[Src::kLut ? 256 : 1];
  const ImgMeta im = imgs[blockIdx.z];
  const int C0 = blockIdx.x * PG_TW, R0 = blockIdx.y * PG_TH;
  if (C0 >= im.w0 || R0 >= im.h0) return;
  const int own_w = min(PG_TW, im.w0 - C0), own_h = min(PG_TH, im.h0 - R0);
  const int last_c = min(PG_TW, im.w0 - 1 - C0), last_r = min(PG_TH, im.h0 - 1 - R0);   // halo included
  if constexpr (Src::kLut) {
    build_rgb8_lut(lut, threadIdx.x);
    __syncthreads();
  }
  const Src src = Src::at(im.src, im.in_w, im.in_h, im.channels, lut);
  const OctMeta& o0 = octs[blockIdx.z * n_oct];
  float* g0 = arena + o0.gauss_off;
  // One working pixel of the staged tile; the column's taps (sy, ry) are the caller's.
  auto stage = [&](int lr, int lc, int sy, float ry) {
    const int r = R0 + lr, c = C0 + lc;
    int sx; float rx;
    bilinear_coef(r, im.ifx, im.in_h, &sx, &rx);
    const float irx = 1.0f - rx, iry = 1.0f - ry;
    float q[12];   // (sx, sy), (sx, sy+1), (sx+1, sy), (sx+1, sy+1), three channels each
    src.fetch(im.in_w, sx, sy, q);
    float v[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      v[ch] = rx * (q[9 + ch] * ry + q[6 + ch] * iry) + irx * (q[3 + ch] * ry + q[ch] * iry);
      tile[ch * SP + lr * SW + lc] = v[ch];
    }
    if (lr < own_h && lc < own_w) {   // the halo belongs to the next tile
      g0[(size_t)r * o0.pitch + c] = (v[0] + v[1] + v[2]) / 3.f;
      if (work) {
        float* dst = work + im.work_off + ((size_t)r * im.w0 + c) * 3;
        dst[0] = v[0]; dst[1] = v[1]; dst[2] = v[2];
      }
    }
  };
  // A thread keeps one column of the tile (its column taps) and walks its rows, PG_ROWS_PER_PASS
  // apart: a warp stores 32 adjacent pixels of a row.  The halo column goes to the last row group,
  // which does not get the halo row (PG_TH + 1 rows).
  constexpr int PG_ROWS_PER_PASS = PG_THREADS / PG_TW;
  static_assert(PG_THREADS % PG_TW == 0 && PG_TW >= PG_TH + 1, "whole row groups; the last one holds the halo column");
  {
    const int lc = threadIdx.x % PG_TW;
    if (lc <= last_c) {
      int sy; float ry;
      bilinear_coef(C0 + lc, im.ify, im.in_w, &sy, &ry);
      for (int lr = threadIdx.x / PG_TW; lr <= last_r; lr += PG_ROWS_PER_PASS) stage(lr, lc, sy, ry);
    }
    const int hr = (int)threadIdx.x - (PG_THREADS - PG_TW);
    if (hr >= 0 && hr <= last_r && PG_TW <= last_c) {
      int sy; float ry;
      bilinear_coef(C0 + PG_TW, im.ify, im.in_w, &sy, &ry);
      stage(hr, PG_TW, sy, ry);
    }
  }
  if (n_oct == 1) return;
  __syncthreads();
  for (int o = 1; o < n_oct; ++o) {
    const OctMeta& om = octs[blockIdx.z * n_oct + o];
    const float ifx = om.ifx, ify = om.ify;
    const int d_r0 = first_tap_at_least(R0, ifx, im.h0, om.h), d_r1 = first_tap_at_least(R0 + PG_TH, ifx, im.h0, om.h);
    const int d_c0 = first_tap_at_least(C0, ify, im.w0, om.w), d_c1 = first_tap_at_least(C0 + PG_TW, ify, im.w0, om.w);
    const int nc = d_c1 - d_c0;
    if (nc == 0) continue;
    float* g = arena + om.gauss_off;
    const int pitch = om.pitch;
    // owned pixels in raster order, PG_THREADS apart: (row, column) steps by (step_r, step_c) with a carry
    const int step_r = PG_THREADS / nc, step_c = PG_THREADS - step_r * nc;
    int dr = d_r0 + (int)threadIdx.x / nc, dc = d_c0 + (int)threadIdx.x % nc;
    for (; dr < d_r1; dr += step_r, dc += step_c) {
      if (dc >= d_c1) { dc -= nc; ++dr; if (dr >= d_r1) break; }
      int sx, sy; float rx, ry;
      bilinear_coef(dr, ifx, im.h0, &sx, &rx);
      bilinear_coef(dc, ify, im.w0, &sy, &ry);
      const float irx = 1.0f - rx, iry = 1.0f - ry;
      const float* p0 = tile + (sx - R0) * SW + (sy - C0);
      const float* p1 = p0 + SW;
      float v[3];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch)
        v[ch] = rx * (p1[ch * SP + 1] * ry + p1[ch * SP] * iry) + irx * (p0[ch * SP + 1] * ry + p0[ch * SP] * iry);
      g[(size_t)dr * pitch + dc] = (v[0] + v[1] + v[2]) / 3.f;
    }
  }
}

// ============================================================ extremum test
// feature/extrema.cc:170-216.  |DoG| (DOGSpace::diff, dog.cc:116-129) is never stored: every
// reader forms it as fabsf(G(s) - G(s+1)) from the Gaussian levels, the reference's value.
// Candidates are appended unordered (one atomic per hit) with a key that encodes the
// canonical order octave -> scale -> raster; k_rank_sort restores that order.
struct ExtremaParams {
  int nscale;
  float pre_color_thres, diff_thres;
  int cap;
  int* cand_count;       // [n_img]
  uint32_t* cand_keys;   // [n_img * cap]
  // tile-perimeter (pixel, scale) pairs whose centre passes pre_color_thres, forwarded by
  // k_blur_extrema to k_extrema_seams; seam_cap bounds every image's perimeter pixels x scales
  int seam_cap;
  int* seam_count;       // [n_img]
  uint32_t* seam_keys;   // [n_img * seam_cap], make_key encoding
};

__device__ __forceinline__ uint32_t make_key(int oct, int scale, int y, int x) {
  return ((uint32_t)oct << 29) | ((uint32_t)scale << 26) | ((uint32_t)y << 13) | (uint32_t)x;
}

// The 26-neighbour test of one pixel at one scale (extrema.cc:177-211).  dog(ds, di, dj) returns
// the |DoG| at scale offset ds, row offset di and column offset dj from the centre.
template <class DoG>
__device__ __forceinline__ bool is_extremum(float center, float pre_color_thres, float diff_thres, const DoG& dog) {
  if (center < pre_color_thres) return false;
  const float cmp1 = center - diff_thres, cmp2 = center + diff_thres;
  bool mx = true, mn = true;
#pragma unroll
  for (int ds = -1; ds <= 1; ++ds) {
#pragma unroll
    for (int di = -1; di <= 1; ++di)
#pragma unroll
      for (int dj = -1; dj <= 1; ++dj) {
        if (ds == 0 && di == 0 && dj == 0) continue;
        const float v = dog(ds, di, dj);
        if (v >= cmp1) mx = false;
        if (v <= cmp2) mn = false;
      }
    if (!mx && !mn) return false;
  }
  return true;
}

__device__ __forceinline__ void append_candidate(const ExtremaParams& ep, int img, uint32_t key) {
  const int slot = atomicAdd(&ep.cand_count[img], 1);
  if (slot < ep.cap) ep.cand_keys[(size_t)img * ep.cap + slot] = key;
}

// ============================================================ K2 blur
// feature/gaussian.hh:29-90 (column pass, then row pass over the column result,
// replicate border, ascending-k mul-then-add), every level from level 0
// (feature/dog.cc:54-57): the grey tile is staged once in shared memory and all
// nlev sigmas are produced from it.
#include "blur_tile.cuh"   // BT_W/BT_H/BT_THREADS, blur_level<C>, TMA + mbarrier helpers

// Any window width; the extrema of its levels are found by k_extrema_scan over every pixel.
__global__ void __launch_bounds__(BT_THREADS)
k_blur_dog(const OctMeta* __restrict__ octs, const int2* __restrict__ span, int n_om,
           float* __restrict__ arena, const __grid_constant__ GaussTable gt) {
  extern __shared__ float smem[];
  const BlurTile tl = find_blur_tile(span, n_om, blockIdx.x);
  const OctMeta om = octs[tl.om];
  const int R = gt.rmax;
  const int GW = BT_W + 2 * R;           // grey tile width
  const int GH = BT_H + 2 * R;
  float* grey = smem;                    // [GH][GW]
  float* colbuf = smem + GH * GW;        // [BT_H][GW]
  const int x0 = tl.tx * BT_W, y0 = tl.ty * BT_H;
  const float* g0 = arena + om.gauss_off;
  const int tid = threadIdx.x;

  for (int i = tid; i < GH * GW; i += BT_THREADS) {
    int yy = i / GW, xx = i - yy * GW;
    int gy = min(max(y0 + yy - R, 0), om.h - 1);
    int gx = min(max(x0 + xx - R, 0), om.w - 1);
    grey[i] = __ldg(g0 + (size_t)gy * om.pitch + gx);
  }
  __syncthreads();

  const int tx = tid & (BT_W - 1), ty = tid / BT_W;   // 64 x 4
  for (int s = 0; s < gt.nlev; ++s) {
    const int c = gt.center[s];
    const float* taps = gt.taps[s];      // taps[k + c], k = -c..c
    const int cw = BT_W + 2 * c;         // columns needed by the row pass
    // column pass
    for (int i = tid; i < BT_H * cw; i += BT_THREADS) {
      int y = i / cw, xx = i - y * cw;
      const float* col = grey + (y + R - c) * GW + (xx + R - c);
      float tmp = 0.f;
      for (int k = 0; k <= 2 * c; ++k) tmp += col[k * GW] * taps[k];
      colbuf[y * GW + xx] = tmp;
    }
    __syncthreads();
    // row pass
    float* lvl = arena + om.gauss_off + (size_t)(s + 1) * om.plane;
#pragma unroll
    for (int i = 0; i < BT_H / 4; ++i) {
      int y = ty + 4 * i;
      const float* row = colbuf + y * GW + tx;
      float tmp = 0.f;
      for (int k = 0; k <= 2 * c; ++k) tmp += row[k] * taps[k];
      int gx = x0 + tx, gy = y0 + y;
      if (gx < om.w && gy < om.h) lvl[(size_t)gy * om.pitch + gx] = tmp;
    }
    __syncthreads();
  }
}

// The reference's defaults (kw = 7 and 13).  PERSISTENT CTAs walk the tile list; the grey
// tile + halo of the NEXT tile is fetched by TMA into the other half of a double buffer
// while this tile's six levels are computed.  TMA zero-fills outside the plane where the
// reference replicates the edge (gaussian.hh:52-58,74-81), so tiles that touch the plane
// border patch their out-of-range cells from the staged in-range ones (the replicated source
// cell is always inside the same staged tile).
//
// The extremum scan is fused in: each level's |DoG| goes to a 3-slot ring of tiles in shared
// memory instead of HBM, and once |DoG| j+1 exists, scale j is tested for the tile's INTERIOR
// pixels (tile rows 1..BT_H-2, columns 1..BT_W-2), whose 26 neighbours all lie in the tile.
// For the tile perimeter it applies the colour threshold only and forwards the few pairs that
// pass to k_extrema_seams.
#define EX_RING_FLOATS (3 * BT_H * BT_W)
__global__ void __launch_bounds__(BT_THREADS, 3)
k_blur_extrema(const OctMeta* __restrict__ octs, const int2* __restrict__ span, int n_om, int n_tiles,
               const TmaDesc* __restrict__ maps, float* __restrict__ arena, const __grid_constant__ GaussTable gt,
               const ExtremaParams ep) {
  extern __shared__ __align__(128) float smem[];
  __shared__ __align__(8) uint64_t s_bar[2];
  __shared__ BlurTile s_tile[2];         // looked up once per tile by thread 0 (binary search)
  const int R = gt.rmax;
  // TMA wants the box origin on a 16-byte boundary of the innermost dimension (a box starting
  // at x0 - 6 faults): the staged tile carries a column halo rounded up to 4 floats.
  const int RX = (R + 3) & ~3;
  const int GW = BT_W + 2 * RX, GH = BT_H + 2 * R;
  const int GSZ = (GH * GW + 31) & ~31;  // floats per grey buffer, 128-byte multiple
  float* grey0 = smem;                   // [2][GH][GW]
  float* colbuf = smem + 2 * GSZ;        // column-pass results as row pairs (blur_tile.cuh)
  float* outT = colbuf + BLUR_COLBUF_FLOATS(6);   // [BT_H][BT_W+1]
  float* ring = outT + BT_H * (BT_W + 1);         // [3][BT_H][BT_W]: |DoG| s in slot s % 3
  const int tid = threadIdx.x;
  const uint32_t tile_bytes = (uint32_t)(GH * GW * sizeof(float));
  int t = blockIdx.x;
  if (tid == 0) {
    sbar_init(sm_u32(&s_bar[0]), 1);
    sbar_init(sm_u32(&s_bar[1]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (t < n_tiles) {
      const BlurTile tl = find_blur_tile(span, n_om, t);
      s_tile[0] = tl;
      sbar_expect_tx(sm_u32(&s_bar[0]), tile_bytes);
      tma_load_2d(sm_u32(grey0), maps + tl.om, tl.tx * BT_W - RX, tl.ty * BT_H - R, sm_u32(&s_bar[0]));
    }
  }
  __syncthreads();
  for (int it = 0; t < n_tiles; t += gridDim.x, ++it) {
    const int b = it & 1;
    float* grey = grey0 + b * GSZ;
    const BlurTile tl = s_tile[b];
    const OctMeta om = octs[tl.om];
    const int x0 = tl.tx * BT_W, y0 = tl.ty * BT_H;
    if (tid == 0 && t + (int)gridDim.x < n_tiles) {
      // the other buffer was last read (and patched) in the previous iteration, which every
      // thread has left through the barrier at the end of the loop body
      const BlurTile nx = find_blur_tile(span, n_om, t + gridDim.x);
      s_tile[b ^ 1] = nx;      // read by everyone after the barrier that ends this iteration
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      sbar_expect_tx(sm_u32(&s_bar[b ^ 1]), tile_bytes);
      tma_load_2d(sm_u32(grey0 + (b ^ 1) * GSZ), maps + nx.om, nx.tx * BT_W - RX, nx.ty * BT_H - R, sm_u32(&s_bar[b ^ 1]));
    }
    sbar_wait(sm_u32(&s_bar[b]), (uint32_t)(it >> 1) & 1u);
    if (x0 - RX < 0 || y0 - R < 0 || x0 + BT_W + RX > om.w || y0 + BT_H + R > om.h) {   // uniform per CTA
      for (int i = tid; i < GH * GW; i += BT_THREADS) {
        const int yy = i / GW, xx = i - yy * GW;
        const int gy = y0 + yy - R, gx = x0 + xx - RX;
        const int cy = min(max(gy, 0), om.h - 1), cx = min(max(gx, 0), om.w - 1);
        if (cy != gy || cx != gx) grey[i] = grey[(cy - y0 + R) * GW + (cx - x0 + RX)];
      }
      __syncthreads();
    }
    const int tx = tid & (BT_W - 1), ty = tid / BT_W;   // 64 x 4
    const int gx = x0 + tx;
    const bool col_in = gx >= 1 && gx <= om.w - 2;      // the reference tests [1, w-2] x [1, h-2]
    const bool col_seam = tx == 0 || tx == BT_W - 1;
    float prev[BT_H / 4];
#pragma unroll
    for (int i = 0; i < BT_H / 4; ++i) prev[i] = grey[(ty + 4 * i + R) * GW + tx + RX];
    for (int s = 0; s < gt.nlev; ++s) {
      if (gt.center[s] == 3) blur_level<3>(grey, colbuf, outT, gt.taps[s], R, RX, GW, tid);
      else blur_level<6>(grey, colbuf, outT, gt.taps[s], R, RX, GW, tid);
      float* lvl = arena + om.gauss_off + (size_t)(s + 1) * om.plane;
      float* dog = ring + (s % 3) * (BT_H * BT_W);
#pragma unroll
      for (int i = 0; i < BT_H / 4; ++i) {
        const int y = ty + 4 * i, gy = y0 + y;
        const float v = outT[y * (BT_W + 1) + tx];
        if (gx < om.w && gy < om.h) lvl[(size_t)gy * om.pitch + gx] = v;
        dog[y * BT_W + tx] = fabsf(prev[i] - v);
        prev[i] = v;
      }
      // The slot written here held |DoG| s-3, last read by the test of scale s-2 in the previous
      // iteration, which every thread has left through the barriers inside blur_level.  No barrier
      // is needed after the writes for the blur either: the next level's column pass touches only
      // grey/colbuf and its row pass (which rewrites outT) sits behind that pass's barrier.
      if (s >= 2) {          // |DoG| s-2, s-1, s are in the ring: test scale j = s-1
        __syncthreads();
        const int j = s - 1;
        const float* d0 = ring + ((s - 2) % 3) * (BT_H * BT_W);
        const float* d1 = ring + ((s - 1) % 3) * (BT_H * BT_W);
        const float* d2 = dog;
#pragma unroll 1       // one copy of the test: the blur kernel is issue-bound, keep its code small
        for (int i = 0; i < BT_H / 4; ++i) {
          const int y = ty + 4 * i, gy = y0 + y;
          if (!col_in || gy < 1 || gy > om.h - 2) continue;
          const int o = y * BT_W + tx;
          const float center = d1[o];
          if (center < ep.pre_color_thres) continue;     // almost every pixel ends here
          if (col_seam || y == 0 || y == BT_H - 1) {
            // tile perimeter: neighbours lie in other tiles, k_extrema_seams finishes the test
            const int slot = atomicAdd(&ep.seam_count[om.img], 1);
            if (slot < ep.seam_cap) ep.seam_keys[(size_t)om.img * ep.seam_cap + slot] = make_key(om.oct, j, gy, gx);
            continue;
          }
          auto at = [&](int ds, int di, int dj) {
            const float* d = ds < 0 ? d0 : ds == 0 ? d1 : d2;
            return d[o + di * BT_W + dj];
          };
          if (is_extremum(center, ep.pre_color_thres, ep.diff_thres, at))
            append_candidate(ep, om.img, make_key(om.oct, j, gy, gx));
        }
      }
    }
    __syncthreads();   // colbuf / outT / the ring / this grey buffer are free for the next tiles
  }
}

// ============================================================ K3 extrema scan
// The 26-neighbour test with |DoG| formed from the Gaussian levels as they are loaded.
//   k_extrema_seams: the (pixel, scale) pairs of tile perimeters (rows 0 and BT_H-1, columns 0
//     and BT_W-1) that k_blur_extrema found above the colour threshold.  Every pixel of the
//     plane lies in exactly one tile, so each pair is tested exactly once.
//   k_extrema_scan: every pixel of every tile, after the generic k_blur_dog.  One CTA per tile.
__device__ __forceinline__ void test_from_levels(const ExtremaParams& ep, const OctMeta& om, const float* arena,
                                                 int j, int gy, int gx, float center) {
  const float* c = arena + om.gauss_off + (size_t)gy * om.pitch + gx;
  auto at = [&](int ds, int di, int dj) {
    const float* q = c + (ptrdiff_t)(j + ds) * om.plane + (ptrdiff_t)di * om.pitch + dj;
    return fabsf(__ldg(q) - __ldg(q + om.plane));
  };
  if (is_extremum(center, ep.pre_color_thres, ep.diff_thres, at))
    append_candidate(ep, om.img, make_key(om.oct, j, gy, gx));
}

__global__ void __launch_bounds__(256)
k_extrema_seams(const OctMeta* __restrict__ octs, int n_oct, const float* __restrict__ arena, const ExtremaParams ep) {
  const int img = blockIdx.y;
  const int n = min(ep.seam_count[img], ep.seam_cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t key = ep.seam_keys[(size_t)img * ep.seam_cap + i];
    const int oct = key >> 29, j = (key >> 26) & 7, gy = (key >> 13) & 8191, gx = key & 8191;
    const OctMeta om = octs[img * n_oct + oct];
    const float* c = arena + om.gauss_off + (size_t)gy * om.pitch + gx;
    test_from_levels(ep, om, arena, j, gy, gx, fabsf(__ldg(c + (size_t)j * om.plane) - __ldg(c + (size_t)(j + 1) * om.plane)));
  }
}

#define EXS_THREADS 192

__global__ void __launch_bounds__(EXS_THREADS, 6)   // latency-bound: many resident CTAs
k_extrema_scan(const OctMeta* __restrict__ octs, const int2* __restrict__ span, int n_om,
               const float* __restrict__ arena, const ExtremaParams ep) {
  const BlurTile tl = find_blur_tile(span, n_om, blockIdx.x);
  const OctMeta om = octs[tl.om];
  const int x0 = tl.tx * BT_W, y0 = tl.ty * BT_H;
  for (int p = threadIdx.x; p < BT_W * BT_H; p += EXS_THREADS) {
    const int gx = x0 + (p & (BT_W - 1)), gy = y0 + p / BT_W;
    if (gx < 1 || gx > om.w - 2 || gy < 1 || gy > om.h - 2) continue;
    const float* c = arena + om.gauss_off + (size_t)gy * om.pitch + gx;
    // Almost every pixel fails the colour threshold at every scale: load the centre's levels
    // 1..nscale-2 together, then test.
    float lv[SIFT_MAX_LEVELS];
#pragma unroll
    for (int l = 1; l < SIFT_MAX_LEVELS; ++l) lv[l] = l <= ep.nscale - 2 ? __ldg(c + (size_t)l * om.plane) : 0.f;
#pragma unroll
    for (int j = 1; j < SIFT_MAX_LEVELS - 1; ++j) {
      if (j >= ep.nscale - 2) break;
      test_from_levels(ep, om, arena, j, gy, gx, fabsf(lv[j] - lv[j + 1]));
    }
  }
}

// ============================================================ K3b ordered compaction
// Rank sort per image: keys are unique, rank = #keys smaller.
__global__ void __launch_bounds__(256)
k_rank_sort(const int* __restrict__ cand_count, const uint32_t* __restrict__ keys,
            uint32_t* __restrict__ sorted, int cap) {
  __shared__ uint32_t sk[1024];
  const int img = blockIdx.y;
  const int n = min(cand_count[img], cap);
  const uint32_t* k = keys + (size_t)img * cap;
  // the grid is sized for a typical count; CTAs stride over the 256-key chunks of the real one
  for (int c0 = blockIdx.x * 256; c0 < n; c0 += gridDim.x * 256) {
    const int i = c0 + threadIdx.x;
    uint32_t mine = i < n ? k[i] : 0xffffffffu;
    int rank = 0;
    for (int base = 0; base < n; base += 1024) {
      int m = min(1024, n - base);
      __syncthreads();
      for (int t = threadIdx.x; t < m; t += blockDim.x) sk[t] = k[base + t];
      __syncthreads();
      for (int t = 0; t < m; ++t) rank += sk[t] < mine;
    }
    if (i < n) sorted[(size_t)img * cap + rank] = mine;
  }
}

// ============================================================ K4 refinement
// Same arithmetic as oracle/small_linalg.h (Eigen FullPivLU restated).
__device__ bool lu3_inverse(const double* a_in, double* inv) {
  double a[9];
  int rowperm[3] = {0, 1, 2}, colperm[3] = {0, 1, 2};
  int nonzero = 3, rank = 0;
  double maxpivot = 0.0;
  for (int i = 0; i < 9; ++i) a[i] = a_in[i];
  for (int k = 0; k < 3; ++k) {
    int br = k, bc = k;
    double big = -1.0;
    for (int i = k; i < 3; ++i)
      for (int j = k; j < 3; ++j) {
        double v = fabs(a[i * 3 + j]);
        if (v > big) { big = v; br = i; bc = j; }
      }
    if (big == 0.0) { nonzero = k; break; }
    if (big > maxpivot) maxpivot = big;
    if (br != k) {
      for (int j = 0; j < 3; ++j) { double w = a[k * 3 + j]; a[k * 3 + j] = a[br * 3 + j]; a[br * 3 + j] = w; }
      int t = rowperm[k]; rowperm[k] = rowperm[br]; rowperm[br] = t;
    }
    if (bc != k) {
      for (int i = 0; i < 3; ++i) { double w = a[i * 3 + k]; a[i * 3 + k] = a[i * 3 + bc]; a[i * 3 + bc] = w; }
      int t = colperm[k]; colperm[k] = colperm[bc]; colperm[bc] = t;
    }
    for (int i = k + 1; i < 3; ++i) a[i * 3 + k] /= a[k * 3 + k];
    for (int i = k + 1; i < 3; ++i)
      for (int j = k + 1; j < 3; ++j) a[i * 3 + j] -= a[i * 3 + k] * a[k * 3 + j];
  }
  double thr = 2.2204460492503131e-16 * 3.0 * maxpivot;
  for (int k = 0; k < nonzero; ++k) if (fabs(a[k * 3 + k]) > thr) ++rank;
  if (rank < 3) return false;
  for (int col = 0; col < 3; ++col) {
    double c[3];
    for (int i = 0; i < 3; ++i) c[i] = rowperm[i] == col ? 1.0 : 0.0;
    c[1] -= a[3] * c[0];
    c[2] -= a[6] * c[0];
    c[2] -= a[7] * c[1];
    c[2] /= a[8];
    c[1] -= a[5] * c[2];
    c[0] -= a[2] * c[2];
    c[1] /= a[4];
    c[0] -= a[1] * c[1];
    c[0] /= a[0];
    for (int i = 0; i < 3; ++i) inv[colperm[i] * 3 + col] = c[i];
  }
  return true;
}

__device__ void sym3_pinv(const double* a_in, double* out) {
  double a[9], v[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 9; ++i) a[i] = a_in[i];
  for (int sweep = 0; sweep < 32; ++sweep) {
    double off = fabs(a[1]) + fabs(a[2]) + fabs(a[5]);
    if (off < 1e-300) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double apq = a[p * 3 + q];
        if (apq == 0.0) continue;
        double theta = (a[q * 3 + q] - a[p * 3 + p]) / (2.0 * apq);
        double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        double c = 1.0 / sqrt(t * t + 1.0);
        double s = t * c;
        for (int k = 0; k < 3; ++k) {
          double akp = a[k * 3 + p], akq = a[k * 3 + q];
          a[k * 3 + p] = c * akp - s * akq;
          a[k * 3 + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {
          double apk = a[p * 3 + k], aqk = a[q * 3 + k];
          a[p * 3 + k] = c * apk - s * aqk;
          a[q * 3 + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          double vkp = v[k * 3 + p], vkq = v[k * 3 + q];
          v[k * 3 + p] = c * vkp - s * vkq;
          v[k * 3 + q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double acc = 0.0;
      for (int k = 0; k < 3; ++k) {
        double l = a[k * 3 + k];
        if (fabs(l) > 1e-6) acc += v[i * 3 + k] * (1.0 / l) * v[j * 3 + k];
      }
      out[i * 3 + j] = acc;
    }
}

struct RefineParams {
  int nscale, depth;
  float offset_thres, contrast_thres, edge_ratio, gauss_sigma, scale_factor;
};

// feature/extrema.cc:63-168: calc_kp_offset(+_iter) and is_edge_response.
__global__ void k_refine(const OctMeta* __restrict__ octs, const float* __restrict__ arena, int n_oct,
                         const int* __restrict__ cand_count, const uint32_t* __restrict__ sorted,
                         RefineParams rp, int cap, pano_sspoint* __restrict__ out, unsigned char* __restrict__ valid) {
  const int img = blockIdx.y;
  const int n = min(cand_count[img], cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
  const size_t slot = (size_t)img * cap + i;
  uint32_t key = sorted[slot];
  int oct = key >> 29, s0 = (key >> 26) & 7, y0 = (key >> 13) & 8191, x0 = key & 8191;
  const OctMeta om = octs[img * n_oct + oct];
  const float* gauss = arena + om.gauss_off;
  const int w = om.w, h = om.h;
  // |DoG| of scale ss: fabsf(G(ss) - G(ss + 1)), as DOGSpace::diff forms it (dog.cc:116-129)
  auto dog_at = [&](int xx, int yy, int ss) {
    const float* q = gauss + (size_t)ss * om.plane + (size_t)yy * om.pitch + xx;
    return fabsf(__ldg(q) - __ldg(q + om.plane));
  };
#define DG(xx, yy, ss) dog_at(xx, yy, ss)
  pano_sspoint sp;
  sp.x = x0; sp.y = y0; sp.pyr_id = oct; sp.scale_id = s0;
  sp.real_x = 0; sp.real_y = 0; sp.dir = 0; sp.scale_factor = 0;
  bool ok = true;
  int nowx = x0, nowy = y0, nows = s0, niter = 0;
  double offset[3] = {0, 0, 0}, delta[3] = {0, 0, 0};
  for (; niter < rp.depth; ++niter) {
    if (!DBETWEEN(nowx, 1, w - 1) || !DBETWEEN(nowy, 1, h - 1) || !DBETWEEN(nows, 1, rp.nscale - 2)) {
      ok = false; break;
    }
    const int x = nowx, y = nowy, s = nows;
    float val = DG(x, y, s);
    delta[0] = (double)((DG(x + 1, y, s) - DG(x - 1, y, s)) / 2);
    delta[1] = (double)((DG(x, y + 1, s) - DG(x, y - 1, s)) / 2);
    delta[2] = (double)((DG(x, y, s + 1) - DG(x, y, s - 1)) / 2);
    double dxx = (double)(DG(x + 1, y, s) + DG(x - 1, y, s) - val - val);
    double dyy = (double)(DG(x, y + 1, s) + DG(x, y - 1, s) - val - val);
    double dss = (double)(DG(x, y, s + 1) + DG(x, y, s - 1) - val - val);
    double dxy = (double)((DG(x + 1, y + 1, s) - DG(x + 1, y - 1, s) - DG(x - 1, y + 1, s) + DG(x - 1, y - 1, s)) / 4);
    double dys = (double)((DG(x, y + 1, s + 1) - DG(x, y - 1, s + 1) - DG(x, y + 1, s - 1) + DG(x, y - 1, s - 1)) / 4);
    double dsx = (double)((DG(x + 1, y, s + 1) - DG(x - 1, y, s + 1) - DG(x + 1, y, s - 1) + DG(x - 1, y, s - 1)) / 4);
    double m[9] = {dxx, dxy, dsx, dxy, dyy, dys, dsx, dys, dss}, inv[9];
    if (!lu3_inverse(m, inv)) sym3_pinv(m, inv);
    for (int q = 0; q < 3; ++q) {
      double acc = inv[q * 3] * delta[0];
      acc += inv[q * 3 + 1] * delta[1];
      acc += inv[q * 3 + 2] * delta[2];
      offset[q] = acc;
    }
    double am = fmax(fabs(offset[0]), fmax(fabs(offset[1]), fabs(offset[2])));
    if (am < (double)rp.offset_thres) break;
    nowx = (int)((double)nowx + round(offset[0]));
    nowy = (int)((double)nowy + round(offset[1]));
    nows = (int)((double)nows + round(offset[2]));
  }
  if (ok && niter == rp.depth) ok = false;
  if (ok) {
    double dextr = offset[0] * delta[0] + offset[1] * delta[1] + offset[2] * delta[2];
    dextr = (double)DG(nowx, nowy, nows) + dextr / 2;
    if (dextr < (double)rp.contrast_thres) ok = false;
  }
  if (ok) {
    sp.x = nowx; sp.y = nowy; sp.scale_id = nows;
    sp.scale_factor = (float)((double)rp.gauss_sigma *
                              pow((double)rp.scale_factor, ((double)nows + offset[2]) / rp.nscale));
    sp.real_x = ((double)nowx + offset[0]) / w;
    sp.real_y = ((double)nowy + offset[1]) / h;
    // is_edge_response on dog[scale_id] at the refined integer position
    const int x = nowx, y = nowy, s = nows;
    float val = DG(x, y, s);
    float dxx = DG(x + 1, y, s) + DG(x - 1, y, s) - val - val;
    float dyy = DG(x, y + 1, s) + DG(x, y - 1, s) - val - val;
    float dxy = (DG(x + 1, y + 1, s) + DG(x - 1, y - 1, s) - DG(x - 1, y + 1, s) - DG(x + 1, y - 1, s)) / 4;
    float det = dxx * dyy - dxy * dxy;
    if (det <= 0) ok = false;
    else {
      float tr2 = (dxx + dyy) * (dxx + dyy);
      float lim = ((rp.edge_ratio + 1) * (rp.edge_ratio + 1)) / rp.edge_ratio;
      if (!(tr2 / det < lim)) ok = false;
    }
  }
#undef DG
  out[slot] = sp;
  valid[slot] = ok ? 1 : 0;
  }
}

// ============================================================ K5 orientation
// feature/orientation.cc:34-100.  Every histogram bin's float sum runs in the reference's
// scan order (xx outer, yy inner), which makes the output bit-identical.
// FOUR LANES per keypoint, eight keypoints per warp: a trip bins four window positions per
// keypoint and adds them to the keypoint's shared-memory histogram one lane after the other —
// lane order is the scan order — so nothing is staged and replayed, and the strictly
// sequential parts (in-place smoothing, the maximum) run for eight keypoints at once instead
// of on one lane of a warp.  Window positions are carried as (xx, yy) per lane instead of a
// divide.
#define ORI_BINS 36
#define ORI_WARPS 4

#define SIFT_MAX_IMG PANO_MAX_SIFT_BATCH   // images per SIFT batch (prefix tables in shared memory)

#define ORI_QUADS 8
__global__ void __launch_bounds__(ORI_WARPS * 32)
k_orientation(const OctMeta* __restrict__ octs, const float* __restrict__ arena, int n_oct, int n_img, int cap,
              const int* __restrict__ cand_count, const pano_sspoint* __restrict__ pts,
              const unsigned char* __restrict__ valid, float ori_radius, int smooth_count,
              int* __restrict__ npeaks, float* __restrict__ dirs, int* __restrict__ work_counter) {
  __shared__ float s_hist[ORI_WARPS][ORI_BINS][ORI_QUADS];   // [bin][quad]: one bank per quad and bin mod 4
  __shared__ uint64_t s_exptab[32];
  __shared__ int s_pref[SIFT_MAX_IMG + 1];      // first flat index of each image's candidates
  load_exp2f_tab(s_exptab, threadIdx.x);
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int i = 0; i < n_img; ++i) { s_pref[i] = acc; acc += min(cand_count[i], cap); }
    s_pref[n_img] = acc;
  }
  __syncthreads();
  const unsigned FULL = 0xffffffffu;
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, l = lane & 3;
  const int total_work = s_pref[n_img];
  float* hist = &s_hist[wid][0][g];             // my keypoint's bin b at hist[b * ORI_QUADS]
  const float halfipi = (float)(0.5 / PANO_PI);   // 0.5f / M_PI evaluated in double
  int img = 0;
  // Candidates are handed out eight at a time from a global counter (most of them were
  // rejected by the refinement and cost nothing; the grid is a few CTAs per SM, not one
  // quad per capacity slot).
  while (true) {
    int flat = 0;
    if (lane == 0) flat = atomicAdd(work_counter, ORI_QUADS);
    flat = __shfl_sync(FULL, flat, 0);
    if (flat >= total_work) break;
    flat += g;
    // ---- per-keypoint constants (identical in the 4 lanes of a quad); rejected candidates get an empty window
    bool live = flat < total_work;
    size_t slot = 0;
    int px = 0, py = 0, w = 0, h = 0, pitch = 0, rad = 0;
    float exp_denom = 1.f;
    const float* lvl = arena;
    if (live) {
      while (flat >= s_pref[img + 1]) ++img;      // indices only grow: resume from the last image
      slot = (size_t)img * cap + (flat - s_pref[img]);
      if (!valid[slot]) {
        if (l == 0) npeaks[slot] = 0;
        live = false;
      } else {
        const pano_sspoint p = pts[slot];
        const OctMeta om = octs[img * n_oct + p.pyr_id];
        lvl = arena + om.gauss_off + (size_t)p.scale_id * om.plane;
        px = p.x; py = p.y; w = om.w; h = om.h; pitch = om.pitch;
        const float gws = p.scale_factor * 1.5f;
        rad = (int)roundf(p.scale_factor * ori_radius);
        exp_denom = 2 * (gws * gws);
      }
    }
    const float fr2 = (float)rad * (float)rad;
    const int side = 2 * rad, total = side * side;
    for (int b = l; b < ORI_BINS; b += 4) hist[b * ORI_QUADS] = 0.f;
    __syncwarp();
    const int total_mx = __reduce_max_sync(FULL, total);
    int xx = -rad, yy = -rad + l;                 // position base + l as (xx, yy), scan order xx outer
    if (side > 0) while (yy >= rad) { yy -= side; ++xx; }
    for (int base = 0; base < total_mx; base += 4) {
      int bin = -1;
      float val = 0.f;
      if (base + l < total) {
        const int newx = px + xx, newy = py + yy;
        if (DBETWEEN(newx, 1, w - 1) && DBETWEEN(newy, 1, h - 1)) {
          const float fx = (float)xx, fy = (float)yy;
          const float d2 = fx * fx + fy * fy;
          if (!(d2 > fr2)) {
            float mag, ort;
            mag_ort_at(lvl, pitch, newx, newy, &mag, &ort);
            int b = (int)roundf((float)ORI_BINS * halfipi * ort);
            if (b == ORI_BINS) b = 0;
            const float weight = glibc_expf(-d2 / exp_denom, s_exptab);
            bin = b;
            val = weight * mag;
          }
        }
        yy += 4;
        while (yy >= rad) { yy -= side; ++xx; }
      }
      // the quad's four positions in scan order
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (l == j && bin >= 0) hist[bin * ORI_QUADS] = hist[bin * ORI_QUADS] + val;
        __syncwarp();
      }
    }
    if (l == 0 && live) {  // in-place sequential smoothing (orientation.cc:70-75)
      for (int K = smooth_count; K--;)
        for (int b = 0; b < ORI_BINS; ++b) {
          float prev = hist[(b == 0 ? ORI_BINS - 1 : b - 1) * ORI_QUADS];
          float next = hist[(b == ORI_BINS - 1 ? 0 : b + 1) * ORI_QUADS];
          hist[b * ORI_QUADS] = (float)((double)hist[b * ORI_QUADS] * 0.5 + (double)(prev + next) * 0.25);
        }
    }
    __syncwarp();
    if (live) {
      float mx = 0.f;
      for (int b = 0; b < ORI_BINS; ++b) if (mx < hist[b * ORI_QUADS]) mx = hist[b * ORI_QUADS];
      const float thres = mx * 0.8f;
      // peaks in ascending bin order: lane l owns bins [9 l, 9 l + 9)
      float my_dir[5];                            // a peak needs two lower neighbours: at most 5 in 9 bins
      int mine = 0;
      for (int b = l * 9; b < l * 9 + 9; ++b) {
        const float hb = hist[b * ORI_QUADS];
        const float prev = hist[(b == 0 ? ORI_BINS - 1 : b - 1) * ORI_QUADS];
        const float next = hist[(b == ORI_BINS - 1 ? 0 : b + 1) * ORI_QUADS];
        if (hb > thres && hb > (prev < next ? next : prev)) {
          double newbin = (double)(float)b - 0.5 + (double)((hb - prev) / (prev + next - 2 * hb));
          if (newbin < 0) newbin += ORI_BINS;
          else if (newbin >= ORI_BINS) newbin -= ORI_BINS;
          const float dir = (float)(newbin / ORI_BINS * 2 * PANO_PI);
          if (mine < 5) my_dir[mine] = dir;
          ++mine;
        }
      }
      // exclusive prefix of the quad's peak counts (live is uniform inside a quad; lanes of dead quads sit out)
      const unsigned qmask = 0xfu << (g * 4);
      int before = 0;
      const int m0 = __shfl_sync(qmask, mine, g * 4 + 0), m1 = __shfl_sync(qmask, mine, g * 4 + 1),
                m2 = __shfl_sync(qmask, mine, g * 4 + 2), m3 = __shfl_sync(qmask, mine, g * 4 + 3);
      if (l > 0) before += m0;
      if (l > 1) before += m1;
      if (l > 2) before += m2;
      for (int k = 0; k < mine && k < 5; ++k)
        if (before + k < SIFT_MAX_PEAKS) dirs[slot * SIFT_MAX_PEAKS + before + k] = my_dir[k];
      if (l == 0) npeaks[slot] = min(m0 + m1 + m2 + m3, SIFT_MAX_PEAKS);
    }
    __syncwarp();
  }
}

// ============================================================ K5b expansion scan
// OrientationAssign::work (orientation.cc:22-32): keypoint order is preserved,
// peaks ascending.  One block per image: exclusive scan of npeaks.
#define SCAN_THREADS 1024
__global__ void __launch_bounds__(SCAN_THREADS)
k_expand_scan(const int* __restrict__ cand_count, const unsigned char* __restrict__ valid,
              const int* __restrict__ npeaks, const float* __restrict__ dirs, int cap,
              int* __restrict__ n_desc, int* __restrict__ n_refined,
              int* __restrict__ desc_cand, float* __restrict__ desc_dir) {
  __shared__ int s_warp[32];
  __shared__ int s_warp2[32];
  const int img = blockIdx.x;
  const int n = min(cand_count[img], cap);
  const int per = (n + SCAN_THREADS - 1) / SCAN_THREADS;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const size_t base = (size_t)img * cap;
  int local = 0, nval = 0;
  for (int k = 0; k < per; ++k) {
    int i = tid * per + k;
    if (i < n && valid[base + i]) { local += npeaks[base + i]; nval++; }
  }
  int incl = local, incl2 = nval;
  for (int d = 1; d < 32; d <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, incl, d);
    int t2 = __shfl_up_sync(0xffffffffu, incl2, d);
    if (lane >= d) { incl += t; incl2 += t2; }
  }
  if (lane == 31) { s_warp[wid] = incl; s_warp2[wid] = incl2; }
  __syncthreads();
  if (wid == 0) {
    int v = s_warp[lane], v2 = s_warp2[lane];
    int a = v, a2 = v2;
    for (int d = 1; d < 32; d <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, a, d);
      int t2 = __shfl_up_sync(0xffffffffu, a2, d);
      if (lane >= d) { a += t; a2 += t2; }
    }
    s_warp[lane] = a - v;   // exclusive
    s_warp2[lane] = a2;     // inclusive (only the last is used)
  }
  __syncthreads();
  int off = s_warp[wid] + incl - local;
  for (int k = 0; k < per; ++k) {
    int i = tid * per + k;
    if (i < n && valid[base + i]) {
      int np = npeaks[base + i];
      for (int q = 0; q < np; ++q) {
        int d = off + q;
        if (d < cap) {
          desc_cand[(size_t)img * cap + d] = i;
          desc_dir[(size_t)img * cap + d] = dirs[(base + i) * SIFT_MAX_PEAKS + q];
        }
      }
      off += np;
    }
  }
  if (tid == SCAN_THREADS - 1) { n_desc[img] = off; n_refined[img] = s_warp2[31]; }
}

// ============================================================ K6 descriptor
// feature/sift.cc:87-152 calc_descriptor, :48-67 trilinear_interpolate, :15-46
// hist_to_descriptor (RootSIFT).  Every bin's float sum runs in the reference's scan order
// (xx outer, yy inner), which makes the output bit-identical.
//   * FOUR LANES per oriented keypoint, eight keypoints per warp.  Lane (ly, lx) of a quad
//     owns the four cells whose row parity is ly and column parity is lx.  A sample adds to
//     the 2x2 block of cells around it — one cell of every parity class — so EVERY record
//     gives every lane of its quad exactly one visit: the walk is balanced by construction,
//     needs no per-cell visit lists (no ballots, no masks, no record buffer) and runs right
//     behind the four records a quad produces per trip.  (One lane per cell keeps only 10 of
//     32 lanes busy: a batch of consecutive scan positions is a few window columns and
//     touches 4-6 of the 16 cells.)
//   * the 32 accumulators a lane owns live in shared memory at bank == lane (conflict-free
//     read-modify-write).  Cells outside the 4x4 grid, rejected positions and idle lanes add
//     +0.0f, which is an exact no-op on these non-negative sums — the walk has no branches.
//   * the window is enumerated by COLUMN INTERVALS (desc_interval.h): the accepted yy of a
//     column form one interval (rotated box ∩ circle ∩ image are convex), so lanes visit only
//     a ~3 % superset of the accepted positions, in scan order, with no compaction ring; the
//     reference's exact tests still decide every position.
// Order of every float sum is the reference's scan order: a quad's records are produced in
// (xx, yy) order, four per trip, and each lane applies them in that order to bins only it
// touches.
#define DESC_WARPS 4
#define DESC_THREADS (DESC_WARPS * 32)

struct DescParams { int hist_scale_factor; int int_factor; };

#define DQ_COLS 96                       // window columns per interval-table block (wider windows take more blocks)

struct __align__(16) DescQuadSmem {
  float acc[32 * 32];                    // [bin * 4 + (cy >> 1) * 2 + (cx >> 1)][lane]
  float r_q[4][32];                      // [record of the trip][reader lane]: weight * wy * wx of the reader's cell (or 0)
  float2 r_h[4][8];                      // [record of the trip][quad]: {hbin - floor(hbin), packed word}
  unsigned char col_len[8][DQ_COLS];     // per quad and table column: interval length ...
  signed char col_y0[8][DQ_COLS];        // ... and first yy
};

#ifndef DESC_MIN_CTAS
#define DESC_MIN_CTAS 6                  // resident CTAs per SM the register allocation is held to
#endif
__global__ void __launch_bounds__(DESC_THREADS, DESC_MIN_CTAS)
k_descriptor(const OctMeta* __restrict__ octs, const ImgMeta* __restrict__ imgs,
             const float* __restrict__ arena, int n_oct, int n_img, int cap,
             const pano_sspoint* __restrict__ pts, const int* __restrict__ n_desc,
             const int* __restrict__ desc_cand, const float* __restrict__ desc_dir,
             DescParams dp, float* __restrict__ out_desc, double* __restrict__ out_coor,
             int* __restrict__ work_counter) {
  extern __shared__ __align__(16) unsigned char desc_smem_raw[];
  __shared__ uint64_t s_exptab[32];
  __shared__ int s_pref[SIFT_MAX_IMG + 1];      // first flat index of each image's descriptors
  load_exp2f_tab(s_exptab, threadIdx.x);
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int i = 0; i < n_img; ++i) { s_pref[i] = acc; acc += min(n_desc[i], cap); }
    s_pref[n_img] = acc;
  }
  __syncthreads();
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int g = lane >> 2, l = lane & 3;        // quad, lane of the quad = record slot of a trip = cell parity class
  DescQuadSmem& S = reinterpret_cast<DescQuadSmem*>(desc_smem_raw)[wid];
  float* const acc = S.acc + lane;              // my 32 accumulators: acc[32 * k]
  const float pi2 = (float)(2 * PANO_PI);
  const float nbin_per_rad = 8 / pi2;
  const float exp_denom = 2 * (4.f * 4.f);
  const int hi_shift = 4 + 2 * l;               // my 2-bit field of the packed word
  const int total = s_pref[n_img];
  // Work is handed out eight descriptors at a time from a global counter: window sizes vary
  // by an order of magnitude with the keypoint scale, and a static assignment left most
  // warps idle while the unlucky ones worked through their heavy keypoints.
  int img = 0;
  while (true) {
    int flat = 0;
    if (lane == 0) flat = atomicAdd(work_counter, 8);
    flat = __shfl_sync(FULL, flat, 0);
    if (flat >= total) break;
    flat += g;
    const bool live = flat < total;               // the last warp-load may have fewer than 8 keypoints

    // ---- per-keypoint constants (identical in the 4 lanes of a quad)
    int px = 0, py = 0, w = 0, h = 0, pitch = 0, radius = 0, side = 0;
    float ort = 0.f, hist_w = 1.f, sinort = 0.f, cosort = 1.f;
    const float* lvl = arena;
    size_t dslot = 0, pslot = 0;
    if (live) {
      while (flat >= s_pref[img + 1]) ++img;      // indices only grow: resume from the last image
      dslot = (size_t)img * cap + (flat - s_pref[img]);
      pslot = (size_t)img * cap + desc_cand[dslot];
      const pano_sspoint p = pts[pslot];
      ort = desc_dir[dslot];
      const OctMeta om = octs[img * n_oct + p.pyr_id];
      lvl = arena + om.gauss_off + (size_t)p.scale_id * om.plane;
      px = p.x; py = p.y; w = om.w; h = om.h; pitch = om.pitch;
      hist_w = p.scale_factor * (float)dp.hist_scale_factor;
      radius = (int)round(PANO_SQRT1_2 * (double)hist_w * (4 + 1));
      glibc_sincosf(ort, &sinort, &cosort);
      side = 2 * radius + 1;
    }
    const float fr2 = (float)radius * (float)radius;
    // conservative bounds on the un-normalised rotated coordinates:
    // bin in [-1,3]  <=>  rot in [-2.5, 1.5] * hist_w (the exact test follows per position)
    const float lo = -2.5f * hist_w - 0.02f * hist_w - 1e-3f, hi = 1.5f * hist_w + 0.02f * hist_w + 1e-3f;
#pragma unroll
    for (int k = 0; k < 32; ++k) acc[32 * k] = 0.f;

    const int side_mx = __reduce_max_sync(FULL, side);
    for (int cb = 0; cb < side_mx; cb += DQ_COLS) {
      // ---- interval table of window columns [cb, cb + DQ_COLS): 4 columns per trip and quad
      int nblk = 0;                               // positions of my keypoint in this block
      const int ncol_mx = min(DQ_COLS, side_mx - cb);
      for (int c0 = 0; c0 < ncol_mx; c0 += 4) {
        const int c = c0 + l;                     // table column; window column cb + c
        int len = 0;
        if (c < DQ_COLS && cb + c < side) {
          int y0, y1;
          desc_col_interval(cb + c - radius, radius, px, py, w, h, sinort, cosort, lo, hi, &y0, &y1);
          len = max(0, y1 - y0 + 1);
          S.col_len[g][c] = (unsigned char)len;
          S.col_y0[g][c] = (signed char)y0;
        }
        len += __shfl_xor_sync(FULL, len, 1);
        len += __shfl_xor_sync(FULL, len, 2);
        nblk += len;
      }
      __syncwarp();
      const int nblk_mx = __reduce_max_sync(FULL, nblk);
      int col = 0, cstart = 0, clen = nblk > 0 ? (int)S.col_len[g][0] : 0;   // my position's column, its first index, its length

      for (int base = 0; base < nblk_mx; base += 4) {
        // ---- one position per lane: the reference's tests and the sample's record
        const int s = base + l;
        float q0 = 0.f, q1 = 0.f, q2 = 0.f, q3 = 0.f, hd = 0.f;
        uint32_t pk = 0;
        if (s < nblk) {
          while (s >= cstart + clen) { cstart += clen; ++col; clen = (int)S.col_len[g][col]; }
          const int xx = cb + col - radius, yy = (int)S.col_y0[g][col] + (s - cstart);
          const int nowx = px + xx, nowy = py + yy;
          const float fx = (float)xx, fy = (float)yy;
          if (DBETWEEN(nowx, 1, w - 1) && DBETWEEN(nowy, 1, h - 1) && !(fx * fx + fy * fy > fr2)) {
            const float y_rot = ((float)(-xx) * sinort + fy * cosort) / hist_w;
            const float x_rot = (fx * cosort + fy * sinort) / hist_w;
            const float ybin = (float)((double)(y_rot + 2.f) - 0.5);
            const float xbin = (float)((double)(x_rot + 2.f) - 0.5);
            if (ybin >= -1.f && ybin <= 3.f && xbin >= -1.f && xbin <= 3.f) {
              float now_mag, now_ort;
              mag_ort_at(lvl, pitch, nowx, nowy, &now_mag, &now_ort);
              float weight = glibc_expf(-(x_rot * x_rot + y_rot * y_rot) / exp_denom, s_exptab);
              weight = weight * now_mag;
              now_ort -= ort;
              if (now_ort < 0) now_ort += pi2;
              if (now_ort > pi2) now_ort -= pi2;
              const float hbin = now_ort * nbin_per_rad;
              const int ybinf = (int)floorf(ybin), xbinf = (int)floorf(xbin), hbinf = (int)floorf(hbin);
              const float yd = ybin - (float)ybinf, xd = xbin - (float)xbinf;
              hd = hbin - (float)hbinf;
              // trilinear_interpolate (sift.cc:48-67): w_y = weight * (dy ? yd : 1 - yd), w_x = w_y * (dx ? xd : 1 - xd).
              // Row parity class 0 / 1 of the 2x2 block: the row with that parity, its factor, or 0 outside the grid.
              const float wy_lo = weight * (1 - yd), wy_hi = weight * yd;    // rows ybinf, ybinf + 1
              const float fx_lo = 1 - xd, fx_hi = xd;                        // columns xbinf, xbinf + 1
              const int yodd = ybinf & 1, xodd = xbinf & 1;                  // parity of the block's first row / column
              // class p takes the first row when its parity matches, the second otherwise
              const int cy0 = ybinf + yodd, cy1 = ybinf + 1 - yodd;          // rows of parity 0 and 1
              const int cx0 = xbinf + xodd, cx1 = xbinf + 1 - xodd;
              const bool vy0 = (unsigned)cy0 <= 3u, vy1 = (unsigned)cy1 <= 3u;
              const bool vx0 = (unsigned)cx0 <= 3u, vx1 = (unsigned)cx1 <= 3u;
              const float wy0 = yodd ? wy_hi : wy_lo, wy1 = yodd ? wy_lo : wy_hi;
              const float fx0 = xodd ? fx_hi : fx_lo, fx1 = xodd ? fx_lo : fx_hi;
              q0 = (vy0 && vx0) ? wy0 * fx0 : 0.f;                           // class (ly, lx) = (0, 0)
              q1 = (vy0 && vx1) ? wy0 * fx1 : 0.f;                           // (0, 1)
              q2 = (vy1 && vx0) ? wy1 * fx0 : 0.f;                           // (1, 0)
              q3 = (vy1 && vx1) ? wy1 * fx1 : 0.f;                           // (1, 1)
              // packed word: hbinf, then per class (cy >> 1) * 2 + (cx >> 1) (0 where the cell is outside: it adds 0)
              const uint32_t hy0 = vy0 ? (uint32_t)(cy0 >> 1) : 0u, hy1 = vy1 ? (uint32_t)(cy1 >> 1) : 0u;
              const uint32_t hx0 = vx0 ? (uint32_t)(cx0 >> 1) : 0u, hx1 = vx1 ? (uint32_t)(cx1 >> 1) : 0u;
              pk = (uint32_t)hbinf | ((hy0 * 2 + hx0) << 4) | ((hy0 * 2 + hx1) << 6) | ((hy1 * 2 + hx0) << 8) | ((hy1 * 2 + hx1) << 10);
            }
          }
        }
        // record l of my quad: reader lane (g, r) finds its factor at r_q[l][g * 4 + r]
        *reinterpret_cast<float4*>(&S.r_q[l][g * 4]) = make_float4(q0, q1, q2, q3);
        S.r_h[l][g] = make_float2(hd, __uint_as_float(pk));
        __syncwarp();
        // ---- the walk: the quad's four records in scan order, my cell of each
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float q = S.r_q[j][lane];
          const float2 hh = S.r_h[j][g];
          const uint32_t word = __float_as_uint(hh.y);
          const float v0 = q * (1 - hh.x), v1 = q * hh.x;
          const uint32_t cell_hi = (word >> hi_shift) & 3u;
          float* a0 = acc + 32 * ((word & 7u) * 4 + cell_hi);
          float* a1 = acc + 32 * (((word + 1u) & 7u) * 4 + cell_hi);
          *a0 = *a0 + v0;
          *a1 = *a1 + v1;
        }
        __syncwarp();
      }
    }

    // ---- RootSIFT: L1 normalise (sequential sum in descriptor order = cell-major), sqrt, * DESC_INT_FACTOR
    __syncwarp();
    const float* qacc = S.acc + g * 4;            // my quad's accumulators: class r at qacc[32 * k + r]
    float sum = 0.f;
    if (l == 0) {
      for (int c = 0; c < 16; ++c) {
        const int cy = c >> 2, cx = c & 3;
        const float* a = qacc + ((cy & 1) * 2 + (cx & 1)) + 32 * ((cy >> 1) * 2 + (cx >> 1));
#pragma unroll
        for (int b = 0; b < 8; ++b) sum += a[32 * 4 * b];
      }
    }
    sum = __shfl_sync(FULL, sum, g * 4);
    if (live) {
      const float fac = (float)dp.int_factor;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int e = l * 4 + 16 * k;             // descriptor elements e .. e+3: cell e >> 3, bins (e & 7) .. +3
        const int c = e >> 3, b = e & 7, cy = c >> 2, cx = c & 3;
        const float* a = qacc + ((cy & 1) * 2 + (cx & 1)) + 32 * ((cy >> 1) * 2 + (cx >> 1));
        float4 o;
        o.x = sqrtf(a[32 * 4 * (b + 0)] / sum) * fac;
        o.y = sqrtf(a[32 * 4 * (b + 1)] / sum) * fac;
        o.z = sqrtf(a[32 * 4 * (b + 2)] / sum) * fac;
        o.w = sqrtf(a[32 * 4 * (b + 3)] / sum) * fac;
        *reinterpret_cast<float4*>(out_desc + dslot * 128 + e) = o;
      }
      if (l == 0) {
        const pano_sspoint p = pts[pslot];
        const ImgMeta im = imgs[img];
        out_coor[dslot * 2] = (p.real_x - 0.5) * im.in_w;
        out_coor[dslot * 2 + 1] = (p.real_y - 0.5) * im.in_h;
        // second half of the coordinate buffer: SSPoint::real_coor, what do_detect_feature returns (sift.cc:150)
        double* out_real = out_coor + (size_t)n_img * cap * 2;
        out_real[dslot * 2] = p.real_x;
        out_real[dslot * 2 + 1] = p.real_y;
      }
    }
    __syncwarp();
  }
}

// ============================================================ host driver
#define PANO_SQRT1_2_HOST 0.70710678118654752440

int host_gauss_kernel(float sigma, int window_factor, float* taps, int cap) {
  // feature/gaussian.cc:17-40 (weights in f32, expf from the host libm: the very
  // function the reference calls)
  int kw = (int)(ceil(0.3 * (sigma / 2 - 1) + 0.8) * window_factor);
  if (kw % 2 == 0) kw++;
  if (kw > cap) return -kw;
  const int center = kw / 2;
  float* k = taps + center;
  k[0] = 1;
  float exp_coeff = (float)(-1.0 / (sigma * sigma * 2)), wsum = 1;
  for (int i = 1; i <= center; i++) {
    k[i] = expf((float)(i * i) * exp_coeff);
    wsum += k[i] * 2;
  }
  float fac = (float)(1.0 / wsum);
  k[0] = fac;
  for (int i = 1; i <= center; i++) { k[i] *= fac; k[-i] = k[i]; }
  return kw;
}

// cuTensorMapEncodeTiled through the runtime's driver-entry-point lookup: the library links
// cudart statically and has no link-time dependency on libcuda.
typedef CUresult (*tma_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int ctx_tma_encode(pano_ctx* ctx, TmaDesc* out, void* base, int rank, const unsigned long long* dims,
                   const unsigned long long* strides_bytes, const unsigned* box) {
  SlowCall sc("ctx_tma_encode");
  if (!ctx->tma_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !fn)
      return ctx_fail(ctx, PANO_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    ctx->tma_encode = fn;
  }
  cuuint64_t gd[5], gs[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
  static_assert(sizeof(TmaDesc) == sizeof(CUtensorMap), "CUtensorMap is 128 bytes");
  CUresult r = ((tma_encode_fn)ctx->tma_encode)((CUtensorMap*)out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, base, gd,
                                                gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return ctx_fail(ctx, PANO_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return PANO_OK;
}

// Everything that shapes a plan: its layout, tables and kernel arguments all follow from these.
static std::vector<int> sift_plan_key(int n, const int* channels, const int* w, const int* h, const pano_params* p,
                                      int cap) {
  static_assert(sizeof(pano_params) % sizeof(int) == 0, "pano_params holds 4-byte fields only");
  std::vector<int> key;
  key.reserve(2 + 3 * (size_t)n + sizeof(pano_params) / sizeof(int));
  key.push_back(n);
  key.push_back(cap);
  for (int i = 0; i < n; ++i) {
    key.push_back(w[i]);
    key.push_back(h[i]);
    key.push_back(channels ? channels[i] : 0);   // 0: f32 source
  }
  const size_t at = key.size();
  key.resize(at + sizeof(pano_params) / sizeof(int));
  memcpy(key.data() + at, p, sizeof(pano_params));
  return key;
}

template <class T>
static int plan_alloc(pano_ctx* ctx, SiftPlan* plan, DevBuf<T>& buf, size_t count) {
  const int rc = buf.alloc(ctx, count);
  if (rc == PANO_OK) {
    auto f = ctx->live.find(buf.get());   // a cached block may be larger than asked for
    plan->bytes += f != ctx->live.end() ? f->second : count * sizeof(T);
  }
  return rc;
}

// A kernel's dynamic shared memory limit belongs to the device, which every context on it shares.  The limit
// set here only grows, so no context launches above a limit another context lowered.
static cudaError_t sift_smem_limit(pano_ctx* ctx, const void* fn, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> set;
  std::lock_guard<std::mutex> lock(mu);
  size_t& cur = set[std::make_pair(ctx->device, fn)];
  if (bytes <= cur) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) cur = bytes;
  return e;
}

int sift_run_batch(pano_ctx* ctx, int n, const void* const* d_src, const int* channels, const int* w, const int* h,
                   const pano_params* p, pano_featureset* fs, std::unique_ptr<SiftWork>* keep, int cap) {
  if (n <= 0 || !d_src || !w || !h || !p || !fs) return ctx_fail(ctx, PANO_ERR_INVALID, "sift: bad argument");
  if (n > SIFT_MAX_IMG) return ctx_fail(ctx, PANO_ERR_INVALID, "sift: %d images in one batch (limit %d): split the batch", n, SIFT_MAX_IMG);
  const int n_oct = p->num_octave, n_scale = p->num_scale;
  if (n_oct < 1 || n_oct > SIFT_MAX_OCT || n_scale < 4 || n_scale - 1 > SIFT_MAX_LEVELS || n_scale - 2 > 7)
    return ctx_fail(ctx, PANO_ERR_INVALID, "sift: NUM_OCTAVE/NUM_SCALE out of supported range");
  if (cap < 256 || cap > SIFT_CAP_MAX) return ctx_fail(ctx, PANO_ERR_INVALID, "sift: list capacity %d out of range", cap);
  {
    // The descriptor kernels keep window columns and offsets in 8 bits: radius <= 127.  A keypoint's
    // scale_factor is GAUSS_SIGMA * SCALE_FACTOR^((s + offset) / nscale) (extrema.cc:99) with
    // 1 <= s <= nscale - 3 and |offset| < OFFSET_THRES (k_refine), its window radius
    // round(sqrt(1/2) * scale_factor * DESC_HIST_SCALE_FACTOR * 5) (sift.cc:100).  The power is monotone
    // in the exponent, so the largest factor sits at one end of the exponent's range.
    const double e_lo = (1.0 - (double)p->offset_thres) / n_scale;
    const double e_hi = (n_scale - 3.0 + (double)p->offset_thres) / n_scale;
    const double sf_max = (double)p->gauss_sigma * std::max(pow((double)p->scale_factor, e_lo), pow((double)p->scale_factor, e_hi));
    const double rad_max = PANO_SQRT1_2_HOST * sf_max * (double)p->desc_hist_scale_factor * 5.0;
    if (!(rad_max <= 127.0))
      return ctx_fail(ctx, PANO_ERR_INVALID, "sift: descriptor windows of up to %.0f pixels radius (limit 127): lower DESC_HIST_SCALE_FACTOR / GAUSS_SIGMA", rad_max);
  }

  // The context's plan serves a batch of the same key.  It is detached while the batch runs, so that an
  // out-of-memory retry inside ctx_alloc cannot free the buffers in use.  A trace (keep) builds a plan of
  // its own and takes its work buffers.
  // Reusing the buffers is safe in stream order only: every reader of the scratch buffers is a kernel of
  // one batch on ctx->stream, queued before the next batch's metadata upload overwrites them.
  std::vector<int> key = sift_plan_key(n, channels, w, h, p, cap);
  std::unique_ptr<SiftPlan> plan;
  if (!keep) {
    plan = std::move(ctx->sift_plan);
    if (plan && plan->key != key) plan.reset();
  }
  const bool fresh = plan == nullptr;

  std::vector<int2> tilespan;     // uploaded when the plan is built
  if (fresh) {
    plan.reset(new SiftPlan);
    plan->key = std::move(key);
    plan->wk.reset(new SiftWork);
    SiftWork* wk = plan->wk.get();
    wk->n_img = n; wk->n_oct = n_oct; wk->n_scale = n_scale; wk->cap = cap;
    wk->h_img.resize(n);
    wk->h_oct.resize((size_t)n * n_oct);
    size_t off = 0;
    int max_w0 = 0, max_h0 = 0;
    int n_tiles = 0;
    size_t seam_cap = 0;            // most tile-perimeter (pixel, scale) pairs of one image
    tilespan.resize((size_t)n * n_oct);
    for (int i = 0; i < n; ++i) {
      if (w[i] < 2 || h[i] < 2) return ctx_fail(ctx, PANO_ERR_INVALID, "sift: image too small");
      if (channels)
        if (int rc = pix8_check(ctx, "sift", i, channels[i], nullptr)) return rc;
      ImgMeta& im = wk->h_img[i];
      im.channels = channels ? channels[i] : 3;
      im.in_w = w[i]; im.in_h = h[i];
      // feature/feature.cc:33-34
      float ratio = p->sift_working_size * 2.0f / (w[i] + h[i]);
      im.h0 = (int)(h[i] * ratio); im.w0 = (int)(w[i] * ratio);
      if (im.w0 < 8 || im.h0 < 8 || im.w0 > 8191 || im.h0 > 8191) return ctx_fail(ctx, PANO_ERR_INVALID, "sift: working size out of range");
      float fx = (float)im.h0 / h[i], fy = (float)im.w0 / w[i];
      im.ifx = 1.f / fx; im.ify = 1.f / fy;
      im.work_off = (long long)off;
      if (keep) off += align_up((size_t)im.w0 * im.h0 * 3, 32);   // the working RGB image, for traces only
      max_w0 = std::max(max_w0, im.w0); max_h0 = std::max(max_h0, im.h0);
      size_t img_tiles = 0;
      for (int o = 0; o < n_oct; ++o) {
        OctMeta& om = wk->h_oct[(size_t)i * n_oct + o];
        om.img = i; om.oct = o;
        if (o == 0) { om.w = im.w0; om.h = im.h0; om.ifx = om.ify = 1.f; }
        else {  // feature/dog.cc:105-107
          float factor = (float)pow((double)p->scale_factor, (double)-o);
          om.w = (int)ceilf(im.w0 * factor); om.h = (int)ceilf(im.h0 * factor);
          if (om.w <= 5 || om.h <= 5) return ctx_fail(ctx, PANO_ERR_INVALID, "sift: octave too small");
          float ofx = (float)om.h / im.h0, ofy = (float)om.w / im.w0;
          om.ifx = 1.f / ofx; om.ify = 1.f / ofy;
        }
        om.pitch = (int)align_up((size_t)om.w, 32);
        om.plane = (long long)om.pitch * om.h;
        om.gauss_off = (long long)off; off += (size_t)om.plane * n_scale;
        tilespan[(size_t)i * n_oct + o] = make_int2(n_tiles, ceil_div(om.w, BT_W));
        n_tiles += ceil_div(om.w, BT_W) * ceil_div(om.h, BT_H);
        img_tiles += (size_t)ceil_div(om.w, BT_W) * ceil_div(om.h, BT_H);
      }
      seam_cap = std::max(seam_cap, img_tiles * (2 * BT_W + 2 * (BT_H - 2)) * (size_t)(n_scale - 3));
    }
    wk->arena_floats = off;
    wk->n_tiles = n_tiles;
    plan->seam_cap = seam_cap;
    plan->max_w0 = max_w0; plan->max_h0 = max_h0;

    GaussTable& gt = plan->gt;
    memset(&gt, 0, sizeof(gt));
    gt.nlev = n_scale - 1;
    {
      float sigma = p->gauss_sigma;  // feature/gaussian.hh:99-102
      for (int s = 0; s < gt.nlev; ++s) {
        int kw = host_gauss_kernel(sigma, p->gauss_window_factor, gt.taps[s], SIFT_MAX_TAPS);
        if (kw < 0) return ctx_fail(ctx, PANO_ERR_INVALID, "sift: gaussian window %d too wide", -kw);
        gt.center[s] = kw / 2;
        gt.rmax = std::max(gt.rmax, kw / 2);
        sigma *= p->scale_factor;
      }
    }
    plan->fast = true;
    for (int s = 0; s < gt.nlev; ++s) plan->fast = plan->fast && (gt.center[s] == 3 || gt.center[s] == 6);
    const int R = gt.rmax;
    if (((size_t)(BT_H + 2 * R) * (BT_W + 2 * R) + (size_t)BT_H * (BT_W + 2 * R)) * sizeof(float) > 200 * 1024)
      return ctx_fail(ctx, PANO_ERR_INVALID, "sift: blur halo too large");

    const size_t nlist = (size_t)n * cap;
    if (int rc = plan_alloc(ctx, plan.get(), wk->arena, off)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->d_img, n)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->d_oct, wk->h_oct.size())) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->d_maps, (size_t)n * n_oct)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->d_tilespan, tilespan.size())) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->cand_count, 2 * n + 2)) return rc;   // [n], [n+1] = work counters, then seam counts
    if (int rc = plan_alloc(ctx, plan.get(), wk->seam_keys, (size_t)n * seam_cap)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->cand_keys, nlist)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->sorted_keys, nlist)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->refined, nlist)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->kp_valid, nlist)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->npeaks, nlist)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->dirs, nlist * SIFT_MAX_PEAKS)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->n_refined, n)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->desc_cand, nlist)) return rc;
    if (int rc = plan_alloc(ctx, plan.get(), wk->desc_dir, nlist)) return rc;
  }
  SiftWork* wk = plan->wk.get();
  const GaussTable& gt = plan->gt;
  const bool fast = plan->fast;
  const size_t seam_cap = plan->seam_cap;
  for (int i = 0; i < n; ++i) wk->h_img[i].src = d_src[i];   // the sources are the one thing a repeat batch changes

  // featureset outputs (per-image capacity `cap`; compact on download)
  const size_t nlist = (size_t)n * cap;
  const int n_om = n * n_oct;
  fs->ctx = ctx; fs->n_images = n; fs->cap = cap;
  if (int rc = fs->d_desc.alloc(ctx, nlist * 128)) return rc;
  if (int rc = fs->d_coor.alloc(ctx, nlist * 4)) return rc;   // scaled coordinates, then real_coor
  fs->d_real = fs->d_coor + nlist * 2;
  if (int rc = fs->d_count.alloc(ctx, n)) return rc;
  fs->base.resize(n);
  for (int i = 0; i < n; ++i) fs->base[i] = (long long)i * cap;

  // metadata upload + counter reset: one launch through the pinned ring (a new plan adds its octave
  // metadata and tile spans, and then its TMA maps)
  {
    void* dsts[4] = {wk->d_img, wk->cand_count, wk->d_oct, wk->d_tilespan};
    const void* srcs[4] = {wk->h_img.data(), nullptr, wk->h_oct.data(), tilespan.data()};
    size_t sizes[4] = {n * sizeof(ImgMeta), (2 * n + 2) * sizeof(int), wk->h_oct.size() * sizeof(OctMeta),
                       tilespan.size() * sizeof(int2)};
    if (int rc = ctx_put_many(ctx, fresh ? 4 : 2, dsts, srcs, sizes)) return rc;
  }
  if (fresh && fast) {
    // one TMA descriptor per grey plane: f32 tensor (w, h), row stride pitch*4, box = tile + halo
    std::vector<TmaDesc> maps(n_om);
    const int R = gt.rmax;
    for (int k = 0; k < n_om; ++k) {
      const OctMeta& om = wk->h_oct[k];
      unsigned long long dims[2] = {(unsigned long long)om.w, (unsigned long long)om.h};
      unsigned long long strides[1] = {(unsigned long long)om.pitch * sizeof(float)};
      unsigned box[2] = {(unsigned)(BT_W + 2 * ((R + 3) & ~3)), (unsigned)(BT_H + 2 * R)};
      if (int rc = ctx_tma_encode(ctx, &maps[k], wk->arena + om.gauss_off, 2, dims, strides, box)) return rc;
    }
    if (int rc = ctx_put(ctx, wk->d_maps, maps.data(), maps.size() * sizeof(TmaDesc))) return rc;
  }

  {
    dim3 g(ceil_div(plan->max_w0, PG_TW), ceil_div(plan->max_h0, PG_TH), n);
    float* work = keep ? wk->arena.get() : nullptr;
    if (int rc = with_reader(src_reader(channels, n), [&](auto tag) -> int {
          using Src = typename decltype(tag)::type;
          PANO_LAUNCH(ctx, src_name<Src>(SRC_NAMES("k_pyramid_grey")), k_pyramid_grey<Src>, g, PG_THREADS, 0,
                      wk->d_img, wk->d_oct, n_oct, wk->arena, work);
          return PANO_OK;
        }))
      return rc;
  }
  {
    const ExtremaParams ep{n_scale, p->pre_color_thres, p->judge_extrema_diff_thres, cap, wk->cand_count, wk->cand_keys,
                           (int)seam_cap, wk->cand_count + n + 2, wk->seam_keys};
    const int R = gt.rmax;
    size_t smem = ((size_t)(BT_H + 2 * R) * (BT_W + 2 * R) + (size_t)BT_H * (BT_W + 2 * R)) * sizeof(float);
    if (fast) {
      // blur + |DoG| + the extremum test of tile interiors in one pass, then the tile seams
      const int GW = BT_W + 2 * ((R + 3) & ~3), GH = BT_H + 2 * R;
      const size_t gsz = ((size_t)GH * GW + 31) & ~(size_t)31;
      size_t smf = (2 * gsz + (size_t)BLUR_COLBUF_FLOATS(6) + (size_t)BT_H * (BT_W + 1) + EX_RING_FLOATS) * sizeof(float);
      PANO_CUDA(ctx, sift_smem_limit(ctx, (const void*)k_blur_extrema, smf));
      const int grid = std::min(wk->n_tiles, ctx->num_sms * 3);
      PANO_LAUNCH(ctx, "k_blur_extrema", k_blur_extrema, grid, BT_THREADS, smf, wk->d_oct, wk->d_tilespan, n_om, wk->n_tiles,
                  wk->d_maps, wk->arena, gt, ep);
      // grid sized for typical counts (a few thousand pairs per image); it strides over the real one
      PANO_LAUNCH(ctx, "k_extrema_seams", k_extrema_seams, dim3(8, n), 256, 0, wk->d_oct, n_oct, wk->arena, ep);
    } else {
      if (smem > 48 * 1024)
        PANO_CUDA(ctx, sift_smem_limit(ctx, (const void*)k_blur_dog, smem));
      PANO_LAUNCH(ctx, "k_blur_dog_generic", k_blur_dog, wk->n_tiles, BT_THREADS, smem, wk->d_oct, wk->d_tilespan, n_om, wk->arena, gt);
      PANO_LAUNCH(ctx, "k_extrema_scan", k_extrema_scan, wk->n_tiles, EXS_THREADS, 0, wk->d_oct, wk->d_tilespan, n_om,
                  wk->arena, ep);
    }
  }
  {
    // latency kernels: grids sized for typical counts (a few thousand candidates per image);
    // they stride over the real device-side count, so nothing is launched per capacity slot
    dim3 g(8, n);
    PANO_LAUNCH(ctx, "k_rank_sort", k_rank_sort, g, 256, 0, wk->cand_count, wk->cand_keys, wk->sorted_keys, cap);
    RefineParams rp{n_scale, p->calc_offset_depth, p->offset_thres, p->contrast_thres, p->edge_ratio,
                    p->gauss_sigma, p->scale_factor};
    dim3 g4(16, n);
    PANO_LAUNCH(ctx, "k_refine", k_refine, g4, 128, 0, wk->d_oct, wk->arena, n_oct, wk->cand_count, wk->sorted_keys, rp, cap,
                wk->refined, wk->kp_valid);
    PANO_LAUNCH(ctx, "k_orientation", k_orientation, ctx->num_sms * 8, ORI_WARPS * 32, 0, wk->d_oct, wk->arena, n_oct, n, cap,
                wk->cand_count, wk->refined, wk->kp_valid, p->ori_radius, p->ori_hist_smooth_count, wk->npeaks, wk->dirs,
                wk->cand_count + n + 1);
    PANO_LAUNCH(ctx, "k_expand_scan", k_expand_scan, n, SCAN_THREADS, 0, wk->cand_count, wk->kp_valid, wk->npeaks,
                wk->dirs, cap, fs->d_count, wk->n_refined, wk->desc_cand, wk->desc_dir);
    DescParams dp{p->desc_hist_scale_factor, p->desc_int_factor};
    const size_t dsm = sizeof(DescQuadSmem) * DESC_WARPS;
    PANO_CUDA(ctx, sift_smem_limit(ctx, (const void*)k_descriptor, dsm));
    const int grid = ctx->num_sms * DESC_MIN_CTAS;
    PANO_LAUNCH(ctx, "k_descriptor", k_descriptor, grid, DESC_THREADS, dsm, wk->d_oct, wk->d_img, wk->arena, n_oct, n, cap,
                wk->refined, fs->d_count, wk->desc_cand, wk->desc_dir, dp, fs->d_desc, fs->d_coor, wk->cand_count + n);
  }
  wk->n_desc = fs->d_count;

  // counts to the host (pinned, async); consumers wait on the completion marker queued behind them
  if (!fs->h_count_pinned.get()) {
    fs->h_count_pinned = ctx_small_pinned_get(ctx, (size_t)2 * n * sizeof(int) + 16);
    if (!fs->h_count_pinned.get()) return ctx_fail(ctx, PANO_ERR_CUDA, "pinned allocation failed");
  }
  {
    int* h_counts = (int*)fs->h_count_pinned.get();
    void* dsts[2] = {h_counts, h_counts + n};
    const void* srcs[2] = {fs->d_count, wk->cand_count};
    size_t sizes[2] = {n * sizeof(int), n * sizeof(int)};
    if (int rc = ctx_store_many(ctx, 2, dsts, srcs, sizes)) return rc;
  }
  PANO_CUDA(ctx, ctx_signal(ctx, &fs->counts_token));
  fs->counts_pending = true;
  fs->counts_on_host = false;

  if (keep) {
    *keep = std::move(plan->wk);
  } else if (ctx->cache_limit && plan->bytes <= ctx->cache_limit) {
    ctx->sift_plan = std::move(plan);
    if (ctx->cached_bytes + ctx->sift_plan->bytes > ctx->cache_limit) ctx_cache_release(ctx, ctx->cache_limit - ctx->sift_plan->bytes);
  }
  return PANO_OK;   // a plan nobody took is freed here
}


// First consumer of a SIFT featureset: waits for the counts.  A list that overflowed its
// capacity (the reference's vectors are unbounded, extrema.cc:56-57) makes the batch run
// again with doubled lists — the sources are still there (pano_b200.h) — and the larger
// capacity becomes this context's starting point.  A failure is sticky.
int featureset_sync_counts(pano_featureset* fs) {
  SlowCall sc("featureset_sync_counts");
  if (fs->error) return fs->error;
  if (fs->counts_on_host) return PANO_OK;
  pano_ctx* ctx = fs->ctx;
  while (fs->counts_pending) {
    cudaError_t e = ctx_wait_signal(ctx, fs->counts_token);
    if (e != cudaSuccess) return fs->error = ctx_cuda(ctx, e, "feature count read-back");
    fs->counts_pending = false;
    const int n = fs->n_images;
    const int* h_counts = (const int*)fs->h_count_pinned.get();
    int worst = 0;
    for (int i = 0; i < n; ++i) worst = std::max(worst, std::max(h_counts[i], h_counts[n + i]));
    if (worst <= fs->cap) {
      fs->h_count.assign(h_counts, h_counts + n);
      break;
    }
    int cap = fs->cap;
    while (cap < worst && cap < SIFT_CAP_MAX) cap *= 2;
    if (cap < worst || fs->src.empty())
      return fs->error = ctx_fail(ctx, PANO_ERR_CAPACITY, "sift: %d list entries in one image exceed the capacity %d", worst, fs->cap);
    // run again with larger lists; the old outputs go back to the pool in stream order
    fs->d_desc.reset(); fs->d_coor.reset(); fs->d_count.reset();
    fs->d_real = nullptr;
    ctx->sift_cap = cap;
    const std::vector<const void*> src = fs->src;
    const std::vector<int> channels = fs->src_channels;
    int rc = sift_run_batch(ctx, n, src.data(), channels.empty() ? nullptr : channels.data(), fs->src_w.data(),
                            fs->src_h.data(), &fs->src_params, fs, nullptr, cap);
    if (rc) return fs->error = rc;
  }
  fs->owned_block.reset();
  fs->counts_on_host = true;
  return PANO_OK;
}
