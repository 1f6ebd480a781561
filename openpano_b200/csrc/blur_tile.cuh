// blur_tile.cuh — the separable Gaussian of the reference (feature/gaussian.hh:29-90: column
// pass first, then the row pass over its result; tmp = 0; tmp += v[k] * tap[k], k ascending,
// separate multiply and add) on one 64x32 tile staged in shared memory, plus the TMA /
// mbarrier helpers that stage the tile.  Shared by the SIFT pyramid (sift.cu) and the
// multi-band blender (blend.cu).
#pragma once
#include "common.cuh"

#define BT_W 64
#define BT_H 32
#define BT_THREADS 256

struct BlurTile { int om; int tx, ty; };

// CTA-level tile index -> (plane entry, tile x, tile y): binary search over the ascending first-tile
// index of the n_om plane entries (the table is a few KB and L1-resident).
// span[k] = (first tile of plane entry k, tiles per tile row)
__device__ __forceinline__ BlurTile find_blur_tile(const int2* __restrict__ span, int n_om, int cta) {
  int lo = 0, hi = n_om - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (span[mid].x <= cta) lo = mid; else hi = mid - 1;
  }
  const int local = cta - span[lo].x, tx_n = span[lo].y;
  BlurTile t;
  t.om = lo; t.ty = local / tx_n; t.tx = local - t.ty * tx_n;
  return t;
}

// Register-blocked passes for compile-time half-widths C (the reference's defaults give kw = 7,
// 13 and, in the blender's last level, 19): both passes keep a sliding window in registers so one
// shared-memory load feeds up to 2C+1 taps, 8 outputs per thread per pass, and work on PAIRS of
// independent outputs (8-byte shared-memory accesses).  Every product is a separately rounded
// multiply (__fmul_rn: never contracted into an FMA with the add that follows).  The arithmetic
// per output is unchanged: tmp = 0; tmp += v[k] * tap[k], k ascending.
//   column pass: thread = (2 adjacent columns) x (8 rows); the staged tile delivers column pairs
//                as one 8-byte load; results go to `colbuf2` as ROW pairs: colbuf2[p][x] =
//                (row 2p, row 2p+1) of column x, row-pair stride `csp` float2 (odd: conflict-free)
//   row pass   : thread = (row pair) x (8 columns), 128 threads; results to `outT` [32][65]
//   store      : lane <-> column, coalesced writes by the caller
// `grey` is the staged tile with a halo of R rows / RX columns (RX a multiple of 4, GW floats per
// row); the column pass covers staged columns [start, start + 2*npair), start = (RX - C) & ~1.
__device__ __forceinline__ float2 fmul2(float2 a, float t) { return make_float2(__fmul_rn(a.x, t), __fmul_rn(a.y, t)); }

#define BLUR_COLBUF_FLOATS(C) (16 * ((((BT_W + 2 * (C) + 2) / 2) * 2) | 1) * 2)   // upper bound for any column parity

template <int C>
__device__ __forceinline__ void blur_level(const float* __restrict__ grey, float* __restrict__ colbuf,
                                           float* __restrict__ outT, const float* __restrict__ taps_g,
                                           int R, int RX, int GW, int tid) {
  constexpr int KW = 2 * C + 1;
  float tap[KW];
#pragma unroll
  for (int k = 0; k < KW; ++k) tap[k] = taps_g[k];
  const int start = (RX - C) & ~1, off = (RX - C) - start;
  const int npair = (BT_W + 2 * C + off + 1) >> 1;
  const int csp = (2 * npair) | 1;
  float2* colbuf2 = reinterpret_cast<float2*>(colbuf);
  // column pass: items = (BT_H/8 row strips) x npair column pairs (<= 256: one round)
  for (int item = tid; item < (BT_H / 8) * npair; item += BT_THREADS) {
    const int strip = item / npair, pr = item - strip * npair;
    const float2* col = reinterpret_cast<const float2*>(grey + (strip * 8 + R - C) * GW + start) + pr;
    const int gw2 = GW >> 1;
    float2 win[8 + 2 * C];
#pragma unroll
    for (int j = 0; j < 8 + 2 * C; ++j) win[j] = col[j * gw2];
#pragma unroll
    for (int r = 0; r < 8; r += 2) {
      float a0x = 0.f, a0y = 0.f, a1x = 0.f, a1y = 0.f;     // rows r and r+1, columns x and x+1
#pragma unroll
      for (int k = 0; k < KW; ++k) {
        const float2 p0 = fmul2(win[r + k], tap[k]);
        const float2 p1 = fmul2(win[r + 1 + k], tap[k]);
        a0x += p0.x; a0y += p0.y; a1x += p1.x; a1y += p1.y;
      }
      float2* dst = colbuf2 + (strip * 4 + (r >> 1)) * csp + 2 * pr;
      dst[0] = make_float2(a0x, a1x);
      dst[1] = make_float2(a0y, a1y);
    }
  }
  __syncthreads();
  // row pass: lane & 15 <-> row pair, (warp, lane >> 4) <-> 8-column strip
  if (tid < 128) {
    const int lane = tid & 31, p = lane & 15, xs = ((tid >> 5) * 2 + (lane >> 4)) * 8;
    const float2* row = colbuf2 + p * csp + off + xs;
    float2 win[8 + 2 * C];
#pragma unroll
    for (int j = 0; j < 8 + 2 * C; ++j) win[j] = row[j];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float ax = 0.f, ay = 0.f;
#pragma unroll
      for (int k = 0; k < KW; ++k) {
        const float2 pp = fmul2(win[c + k], tap[k]);
        ax += pp.x; ay += pp.y;
      }
      outT[(2 * p) * (BT_W + 1) + xs + c] = ax;
      outT[(2 * p + 1) * (BT_W + 1) + xs + c] = ay;
    }
  }
  __syncthreads();
}

// ---- TMA / mbarrier helpers (tile loads of the blur kernel)
__device__ __forceinline__ uint32_t sm_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void sbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sbar_wait(uint32_t bar, uint32_t parity) {   // bounded: a protocol bug traps
  uint32_t done = 0;
  for (uint32_t spin = 0; spin < (1u << 28); ++spin) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) return;
  }
  __trap();
}
// 2-D tiled TMA load (cp.async.bulk.tensor): box origin (cx, cy) may lie outside the tensor,
// out-of-range elements arrive as zeros.  The descriptor lives in global memory (written by
// an earlier kernel of this stream), hence the tensormap-proxy acquire fence.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const TmaDesc* map, int cx, int cy, uint32_t bar) {
  asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(map) : "memory");
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(map), "r"(cx), "r"(cy), "r"(bar) : "memory");
}

