// ransac.cu — RANSAC inlier scoring on the device (SURVEY.md §8f.1).
//
// Replaces the scoring half of TransformEstimation::get_transform (stitch/transform_estimate.cc
// :68-85): for every hypothesis of every image pair, get_inliers (:132-148) counts the matches
// whose transferred point lies within the inlier distance; the first hypothesis with the largest
// count wins (update_max is a strict <, lib/utils.hh:58-63) and its inlier set is returned.
// 1500 hypotheses x ~1000 matches x hundreds of pairs are independent evaluations; hypothesis
// generation (random sampling + normalised DLT, :89-130) stays host geometry with the caller's
// seed policy.  The arithmetic is the reference's: f64, the three-term products summed in index
// order, idenom = 1.f / z, strict < against the float threshold squared.
#include "common.cuh"
#include <string.h>
#include <vector>

struct RansacPair {
  long long match_off, hyp_off;
  int n_match, n_hyp;
  float inlier_dist;
  int pad;
};

__device__ __forceinline__ bool ransac_inlier(const double* __restrict__ h, double2 p2, double2 p1, float inlier_dist) {
  double z = p2.x * h[6]; z += p2.y * h[7]; z += 1.0 * h[8];
  double x = p2.x * h[0]; x += p2.y * h[1]; x += 1.0 * h[2];
  double y = p2.x * h[3]; y += p2.y * h[4]; y += 1.0 * h[5];
  const double idenom = (double)1.f / z;
  const double dx = x * idenom - p1.x, dy = y * idenom - p1.y;
  const double dist = dx * dx + dy * dy;
  return dist < (double)inlier_dist;
}

// one warp per hypothesis: lanes stride over the pair's matches; pairs on gridDim.y (at most 65,535:
// the blocks of a y index take every gridDim.y-th pair)
__global__ void __launch_bounds__(256)
k_ransac_count(const RansacPair* __restrict__ pairs, int n_pairs, const double2* __restrict__ kp1,
               const double2* __restrict__ kp2, const double* __restrict__ homos, int* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  for (int p = blockIdx.y; p < n_pairs; p += gridDim.y) {
    const RansacPair pr = pairs[p];
    for (int k = blockIdx.x * 8 + (threadIdx.x >> 5); k < pr.n_hyp; k += gridDim.x * 8) {
      double h[9];
#pragma unroll
      for (int q = 0; q < 9; ++q) h[q] = __ldg(homos + (pr.hyp_off + k) * 9 + q);
      int cnt = 0;
      for (int i = lane; i < pr.n_match; i += 32)
        cnt += ransac_inlier(h, kp2[pr.match_off + i], kp1[pr.match_off + i], pr.inlier_dist) ? 1 : 0;
      for (int off = 16; off; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
      if (lane == 0) counts[pr.hyp_off + k] = cnt;
    }
  }
}

// one CTA per pair: first hypothesis with the largest count, then its inlier flags
__global__ void __launch_bounds__(256)
k_ransac_select(const RansacPair* __restrict__ pairs, const double2* __restrict__ kp1, const double2* __restrict__ kp2,
                const double* __restrict__ homos, const int* __restrict__ counts, int* __restrict__ best_hyp,
                int* __restrict__ best_count, unsigned char* __restrict__ flags) {
  __shared__ long long s_key[8];
  __shared__ int s_best;
  const RansacPair pr = pairs[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31;
  // key = count * 2^32 + (2^31 - 1 - index): the maximum is the largest count, lowest index
  long long key = -1;
  for (int k = tid; k < pr.n_hyp; k += 256) {
    const long long c = ((long long)counts[pr.hyp_off + k] << 32) | (unsigned)(0x7fffffff - k);
    key = c > key ? c : key;
  }
  for (int off = 16; off; off >>= 1) { const long long o = __shfl_xor_sync(0xffffffffu, key, off); key = o > key ? o : key; }
  if (lane == 0) s_key[tid >> 5] = key;
  __syncthreads();
  if (tid == 0) {
    for (int q = 1; q < 8; ++q) key = s_key[q] > key ? s_key[q] : key;
    const int b = key < 0 ? -1 : 0x7fffffff - (int)(key & 0xffffffffLL);
    s_best = b;
    best_hyp[blockIdx.x] = b;
    best_count[blockIdx.x] = key < 0 ? 0 : (int)(key >> 32);
  }
  __syncthreads();
  const int b = s_best;
  double h[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) h[q] = b < 0 ? 0.0 : __ldg(homos + (pr.hyp_off + b) * 9 + q);
  for (int i = tid; i < pr.n_match; i += 256)
    flags[pr.match_off + i] = (b >= 0 && ransac_inlier(h, kp2[pr.match_off + i], kp1[pr.match_off + i], pr.inlier_dist)) ? 1 : 0;
}

extern "C" int pano_ransac_score_pairs(pano_ctx* ctx, int n_pairs, const pano_ransac_pair* pairs, int* best_hyp,
                                       int* best_count, int* const* hyp_counts, unsigned char* const* inlier_flags) {
  ctx_enter(ctx);
  if (!ctx || n_pairs < 0 || (n_pairs && (!pairs || !best_hyp || !best_count))) return PANO_ERR_INVALID;
  if (n_pairs == 0) return PANO_OK;
  std::vector<RansacPair> meta(n_pairs);
  long long nm = 0, nh = 0;
  int max_hyp = 0;
  for (int k = 0; k < n_pairs; ++k) {
    const pano_ransac_pair& p = pairs[k];
    if (p.n_match < 0 || p.n_hyp < 0 || (p.n_match && (!p.kp1_xy || !p.kp2_xy)) || (p.n_hyp && !p.homos))
      return ctx_fail(ctx, PANO_ERR_INVALID, "ransac: pair %d has a null or negative field", k);
    meta[k] = RansacPair{nm, nh, p.n_match, p.n_hyp, p.inlier_thres * p.inlier_thres, 0};   // sqr(float), utils.hh:25
    nm += p.n_match; nh += p.n_hyp;
    max_hyp = std::max(max_hyp, p.n_hyp);
  }
  // host staging: one pinned block, three async copies
  const size_t b_kp = (size_t)nm * 2 * sizeof(double), b_h = (size_t)nh * 9 * sizeof(double);
  const size_t b_meta = (size_t)n_pairs * sizeof(RansacPair);
  const size_t b_out = (size_t)nh * sizeof(int) + (size_t)2 * n_pairs * sizeof(int) + (size_t)nm;
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));            // the staging buffers may still feed earlier copies
  char* st = (char*)ctx_pinned(ctx, 2 * b_kp + b_h + b_meta + 64);
  char* so = (char*)ctx_pinned2(ctx, b_out + 64);
  if (!st || !so) return ctx_fail(ctx, PANO_ERR_CUDA, "ransac: pinned staging allocation failed");
  double* s1 = (double*)st; double* s2 = (double*)(st + b_kp); double* sh = (double*)(st + 2 * b_kp);
  for (int k = 0; k < n_pairs; ++k) {
    const pano_ransac_pair& p = pairs[k];
    if (p.n_match) {
      memcpy(s1 + meta[k].match_off * 2, p.kp1_xy, (size_t)p.n_match * 16);
      memcpy(s2 + meta[k].match_off * 2, p.kp2_xy, (size_t)p.n_match * 16);
    }
    if (p.n_hyp) memcpy(sh + meta[k].hyp_off * 9, p.homos, (size_t)p.n_hyp * 72);
  }
  memcpy(st + 2 * b_kp + b_h, meta.data(), b_meta);
  DevBuf<char> d_in, d_out;
  int rc = d_in.alloc(ctx, 2 * b_kp + b_h + b_meta + 64);
  if (!rc) rc = d_out.alloc(ctx, b_out + 64);
  if (rc) return rc;
  PANO_CUDA(ctx, cudaMemcpyAsync(d_in, st, 2 * b_kp + b_h + b_meta, cudaMemcpyHostToDevice, ctx->stream));
  const double2* d_kp1 = (const double2*)d_in.get(); const double2* d_kp2 = (const double2*)(d_in + b_kp);
  const double* d_h = (const double*)(d_in + 2 * b_kp);
  const RansacPair* d_meta = (const RansacPair*)(d_in + 2 * b_kp + b_h);
  int* d_counts = (int*)d_out.get(); int* d_best = d_counts + nh; int* d_bcnt = d_best + n_pairs;
  unsigned char* d_flags = (unsigned char*)(d_bcnt + n_pairs);
  dim3 grid((unsigned)std::max(1, std::min((max_hyp + 7) / 8, 64)), grid_y(n_pairs));
  PANO_LAUNCH(ctx, "k_ransac_count", k_ransac_count, grid, 256, 0, d_meta, n_pairs, d_kp1, d_kp2, d_h, d_counts);
  PANO_LAUNCH(ctx, "k_ransac_select", k_ransac_select, n_pairs, 256, 0, d_meta, d_kp1, d_kp2, d_h, d_counts, d_best, d_bcnt,
              d_flags);
  PANO_CUDA(ctx, cudaMemcpyAsync(so, d_out, b_out, cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const int* h_counts = (const int*)so;
  const int* h_best = h_counts + nh;
  const int* h_bcnt = h_best + n_pairs;
  const unsigned char* h_flags = (const unsigned char*)(h_bcnt + n_pairs);
  for (int k = 0; k < n_pairs; ++k) {
    best_hyp[k] = h_best[k]; best_count[k] = h_bcnt[k];
    if (hyp_counts && hyp_counts[k] && pairs[k].n_hyp) memcpy(hyp_counts[k], h_counts + meta[k].hyp_off, (size_t)pairs[k].n_hyp * sizeof(int));
    if (inlier_flags && inlier_flags[k] && pairs[k].n_match) memcpy(inlier_flags[k], h_flags + meta[k].match_off, (size_t)pairs[k].n_match);
  }
  return PANO_OK;
}
